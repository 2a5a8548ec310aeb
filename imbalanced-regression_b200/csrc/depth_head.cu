// NYUD2-DIR's depth head (nyud2-dir/models/modules.py:145, 169: R.conv2 = nn.Conv2d(c, 1, 5, stride 1, padding 2,
// bias)) as three memory-bound kernels over the NHWC bf16 feature map x [n, h, w, c]; the weight is the reference's fp32
// [1, c, 5, 5] tensor as it is.
//
//   fwd    y[p]        = b + sum_{ch, tap} w[ch, tap] * x[p + tap - 2, ch]     fp32 [n, h, w, 1]
//   dgrad  dx[p, ch]   = sum_tap w[ch, tap] * dy[p - tap + 2]                  bf16 [n, h, w, c]
//   wgrad  dw[ch, tap] = sum_p dy[p] * x[p + tap - 2, ch],  db = sum_p dy[p]   fp32, overwritten
//
// All three walk the same 16 x 32 pixel tiles with a 2-pixel halo staged in shared memory (zeros outside the image).
// Every sum has a fixed order that depends on nothing but the pixel / output it produces, and there are no atomics:
//   fwd    per pixel: channel groups of 8 ascending, then ky, kx, channel; the bias added last.
//   dgrad  per (pixel, channel): taps (ky, kx) ascending.
//   wgrad  per tile: dw over columns left to right within a tile row, then tile rows top to bottom; db over a fixed
//          split of the tile's pixels across 32 lanes and a butterfly (dy = 0 outside the image); then the per-tile
//          partials in tile order, in a second launch.
#include "common.cuh"

namespace dirb200 {
namespace {

constexpr int TH = 16, TW = 32;                    // output tile
constexpr int HR = TH + 4, HC = TW + 4;            // halo tile
constexpr int XROW = HC * 16 + 16;                 // bytes per halo row of one 8-channel group, +16: the 8 lanes of a
                                                   // quarter warp read 8 different rows without a bank conflict

__device__ __forceinline__ void bf16x8_to_f32(const uint4 u, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 v = __bfloat1622float2(h[i]);
    f[2 * i] = v.x;
    f[2 * i + 1] = v.y;
  }
}

struct Tile {
  int b, y0, x0;
};
__device__ __forceinline__ Tile tile_of(int t, int h, int w) {
  const int tx = (w + TW - 1) / TW, ty = (h + TH - 1) / TH;
  Tile r;
  r.x0 = (t % tx) * TW;
  t /= tx;
  r.y0 = (t % ty) * TH;
  r.b = t / ty;
  return r;
}

// the halo rows / columns of 8 channels (group g) of a tile -> xs [HR][XROW bytes]
__device__ __forceinline__ void stage_x(const __nv_bfloat16* __restrict__ x, const Tile& t, int h, int w, int c, int g,
                                        unsigned char* xs, int tid, int nthreads) {
  for (int i = tid; i < HR * HC; i += nthreads) {
    const int r = i / HC, cc = i % HC;
    const int yy = t.y0 - 2 + r, xx = t.x0 - 2 + cc;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (yy >= 0 && yy < h && xx >= 0 && xx < w)
      v = *reinterpret_cast<const uint4*>(x + ((static_cast<int64_t>(t.b) * h + yy) * w + xx) * c + g * 8);
    *reinterpret_cast<uint4*>(xs + r * XROW + cc * 16) = v;
  }
}

// w [c][25] fp32 -> ws [25][c] (tap-major: 8 consecutive channels of a tap are two float4)
__device__ __forceinline__ void stage_w(const float* __restrict__ wt, int c, float* ws, int tid, int nthreads) {
  for (int i = tid; i < 25 * c; i += nthreads) ws[(i % 25) * c + i / 25] = wt[i];
}

// ---------------------------------------------------------------------------------------------------- forward
// 128 threads: thread (s, r) = (tid / 16, tid % 16) computes the 4 pixels (r, 4s .. 4s + 3) of the tile.
__global__ void __launch_bounds__(128)
depth_head_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ wt, const float* __restrict__ bias,
                      float* __restrict__ y, int h, int w, int c) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned char* xs = smem;
  float* ws = reinterpret_cast<float*>(smem + HR * XROW);
  const int tid = threadIdx.x;
  const Tile t = tile_of(blockIdx.x, h, w);
  const int r = tid % 16, s = tid / 16;
  stage_w(wt, c, ws, tid, 128);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int g = 0; g < c / 8; ++g) {
    __syncthreads();                                     // previous group's reads (and the weights' writes) done
    stage_x(x, t, h, w, c, g, xs, tid, 128);
    __syncthreads();
#pragma unroll 1
    for (int ky = 0; ky < 5; ++ky) {
      float xv[8][8];
#pragma unroll
      for (int k = 0; k < 8; ++k)
        bf16x8_to_f32(*reinterpret_cast<const uint4*>(xs + (r + ky) * XROW + (4 * s + k) * 16), xv[k]);
#pragma unroll
      for (int kx = 0; kx < 5; ++kx) {
        const float4 w0 = *reinterpret_cast<const float4*>(ws + (ky * 5 + kx) * c + g * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(ws + (ky * 5 + kx) * c + g * 8 + 4);
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[p] = fmaf(wv[j], xv[p + kx][j], acc[p]);
      }
    }
  }
  const int yy = t.y0 + r;
  if (yy >= h) return;
  const float b = bias[0];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int xx = t.x0 + 4 * s + p;
    if (xx < w) y[(static_cast<int64_t>(t.b) * h + yy) * w + xx] = acc[p] + b;
  }
}

// ---------------------------------------------------------------------------------------------------- dgrad
// 256 threads; work item = (4-pixel row segment, channel group of 8), the group fastest so that the lanes of a warp
// store consecutive 16-byte pieces of one pixel.
__global__ void __launch_bounds__(256)
depth_head_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ wt, __nv_bfloat16* __restrict__ dx,
                        int h, int w, int c) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* ds = reinterpret_cast<float*>(smem);            // [HR][HC]: dy at (y0 - 2 + r, x0 - 2 + cc)
  float* ws = ds + HR * HC;
  const int tid = threadIdx.x;
  const Tile t = tile_of(blockIdx.x, h, w);
  stage_w(wt, c, ws, tid, 256);
  for (int i = tid; i < HR * HC; i += 256) {
    const int r = i / HC, cc = i % HC;
    const int yy = t.y0 - 2 + r, xx = t.x0 - 2 + cc;
    ds[i] = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? dy[(static_cast<int64_t>(t.b) * h + yy) * w + xx] : 0.f;
  }
  __syncthreads();
  const int groups = c / 8;
  for (int item = tid; item < TH * (TW / 4) * groups; item += 256) {
    const int g = item % groups, seg = item / groups;
    const int r = seg / (TW / 4), s = seg % (TW / 4);
    const int yy = t.y0 + r;
    if (yy >= h || t.x0 + 4 * s >= w) continue;
    float acc[4][8];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[p][j] = 0.f;
#pragma unroll
    for (int ky = 0; ky < 5; ++ky) {
      // dx at column 4s + p gathers dy at halo column 4s + p + 4 - kx, halo row r + 4 - ky
      float dv[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) dv[k] = ds[(r + 4 - ky) * HC + 4 * s + k];
#pragma unroll
      for (int kx = 0; kx < 5; ++kx) {
        const float4 w0 = *reinterpret_cast<const float4*>(ws + (ky * 5 + kx) * c + g * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(ws + (ky * 5 + kx) * c + g * 8 + 4);
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(wv[j], dv[p + 4 - kx], acc[p][j]);
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int xx = t.x0 + 4 * s + p;
      if (xx >= w) break;
      uint4 u;
      __nv_bfloat162* hv = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) hv[i] = __floats2bfloat162_rn(acc[p][2 * i], acc[p][2 * i + 1]);
      *reinterpret_cast<uint4*>(dx + ((static_cast<int64_t>(t.b) * h + yy) * w + xx) * c + g * 8) = u;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- wgrad
// One CTA per (tile, channel group of 8): 80 of its 96 threads, (ky, r) = (tid / 16, tid % 16), sum over tile row r
// the 5 x 8 products dy[p] * x[p + (ky, kx) - 2, ch] for kx = 0..4 (a sliding window of 5 halo pixels in registers);
// the 16 row sums are then added in row order.  part[tile][ch * 25 + tap]; db_part[tile] = the tile's sum of dy
// (channel group 0 only).
constexpr int WG_THREADS = 96;
constexpr int DYROW = TW + 1;                          // padded: 8 lanes on 8 rows hit 8 banks

__global__ void __launch_bounds__(WG_THREADS)
depth_head_wgrad_partial_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ dy,
                                float* __restrict__ part, float* __restrict__ db_part, int h, int w, int c) {
  __shared__ __align__(16) unsigned char xs[HR * XROW];
  __shared__ float ds[TH * DYROW];
  __shared__ float red[5 * TH * 40];
  const int tid = threadIdx.x;
  const Tile t = tile_of(blockIdx.x, h, w);
  const int g = blockIdx.y;
  stage_x(x, t, h, w, c, g, xs, tid, WG_THREADS);
  for (int i = tid; i < TH * TW; i += WG_THREADS) {
    const int r = i / TW, cc = i % TW;
    const int yy = t.y0 + r, xx = t.x0 + cc;
    ds[r * DYROW + cc] = (yy < h && xx < w) ? dy[(static_cast<int64_t>(t.b) * h + yy) * w + xx] : 0.f;
  }
  __syncthreads();
  if (tid < 5 * TH) {
    const int ky = tid / TH, r = tid % TH;
    const unsigned char* row = xs + (r + ky) * XROW;
    float acc[5][8];
#pragma unroll
    for (int kx = 0; kx < 5; ++kx)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[kx][j] = 0.f;
    float win[5][8];                                   // halo columns px .. px + 4
#pragma unroll
    for (int k = 0; k < 4; ++k) bf16x8_to_f32(*reinterpret_cast<const uint4*>(row + k * 16), win[k]);
#pragma unroll
    for (int px = 0; px < TW; ++px) {
      bf16x8_to_f32(*reinterpret_cast<const uint4*>(row + (px + 4) * 16), win[(px + 4) % 5]);
      const float d = ds[r * DYROW + px];
#pragma unroll
      for (int kx = 0; kx < 5; ++kx)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[kx][j] = fmaf(d, win[(px + kx) % 5][j], acc[kx][j]);
    }
#pragma unroll
    for (int kx = 0; kx < 5; ++kx)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[(ky * TH + r) * 40 + kx * 8 + j] = acc[kx][j];
  }
  __syncthreads();
  for (int o = tid; o < 200; o += WG_THREADS) {          // o = ky * 40 + kx * 8 + j
    const int ky = o / 40, kx = (o % 40) / 8, j = o % 8;
    float s = 0.f;
    for (int r = 0; r < TH; ++r) s += red[(ky * TH + r) * 40 + kx * 8 + j];
    part[static_cast<int64_t>(blockIdx.x) * 25 * c + (g * 8 + j) * 25 + ky * 5 + kx] = s;
  }
  if (g == 0 && tid < 32) {
    float s = 0.f;
    for (int i = tid; i < TH * TW; i += 32) s += ds[(i / TW) * DYROW + i % TW];
    s = warp_sum(s);
    if (tid == 0) db_part[blockIdx.x] = s;
  }
}

// out[k] = sum over tiles, in tile order, of part[tile][k] (k < 25c: dw), and db = the same over db_part
__global__ void __launch_bounds__(256)
depth_head_wgrad_reduce_kernel(const float* __restrict__ part, const float* __restrict__ db_part, int tiles, int k_total,
                               float* __restrict__ dw, float* __restrict__ db) {
  const int k = blockIdx.x * 256 + threadIdx.x;
  if (k > k_total) return;
  const float* src = k < k_total ? part + k : db_part;
  const int64_t stride = k < k_total ? k_total : 1;
  float s = 0.f;
#pragma unroll 8
  for (int i = 0; i < tiles; ++i) s += src[i * stride];
  if (k < k_total) dw[k] = s;
  else db[0] = s;
}

int tiles_of(int n, int h, int w) { return n * ((h + TH - 1) / TH) * ((w + TW - 1) / TW); }

bool shape_ok(int n, int h, int w, int c, const char* who) {
  if (!(c >= 8 && c <= 256 && c % 8 == 0)) {
    set_error("%s: c must be a multiple of 8 from 8 to 256 (got %d)", who, c);
    return false;
  }
  if (!(n > 0 && h > 0 && w > 0)) {
    set_error("%s: n, h and w must be positive (got %d, %d, %d)", who, n, h, w);
    return false;
  }
  if (static_cast<int64_t>(n) * h * w * c >= (int64_t(1) << 31)) {
    set_error("%s: n * h * w * c must be below 2^31", who);
    return false;
  }
  return true;
}

size_t wgrad_ws_bytes(int n, int h, int w, int c) {
  return static_cast<size_t>(tiles_of(n, h, w)) * (25 * static_cast<size_t>(c) + 1) * sizeof(float);
}

}  // namespace
}  // namespace dirb200

using namespace dirb200;

extern "C" {

int dirb200_depth_head_fwd(const void* x, const float* w, const float* b, float* y, int n, int h, int wd, int c,
                           void* stream) {
  if (!shape_ok(n, h, wd, c, "depth_head_fwd")) return DIRB200_ERR_ARG;
  DIRB_CHECK_ARG(x && w && b && y, "depth_head_fwd: null pointer");
  const size_t smem = HR * XROW + 25 * static_cast<size_t>(c) * sizeof(float);
  depth_head_fwd_kernel<<<tiles_of(n, h, wd), 128, smem, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(x), w, b,
                                                                              y, h, wd, c);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_depth_head_dgrad(const float* dy, const float* w, void* dx, int n, int h, int wd, int c, void* stream) {
  if (!shape_ok(n, h, wd, c, "depth_head_dgrad")) return DIRB200_ERR_ARG;
  DIRB_CHECK_ARG(dy && w && dx, "depth_head_dgrad: null pointer");
  const size_t smem = (HR * HC + 25 * static_cast<size_t>(c)) * sizeof(float);
  depth_head_dgrad_kernel<<<tiles_of(n, h, wd), 256, smem, as_stream(stream)>>>(dy, w, static_cast<__nv_bfloat16*>(dx),
                                                                                h, wd, c);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

size_t dirb200_depth_head_wgrad_workspace_bytes(int n, int h, int wd, int c) {
  if (!shape_ok(n, h, wd, c, "depth_head_wgrad_workspace_bytes")) return 0;
  return wgrad_ws_bytes(n, h, wd, c);
}

int dirb200_depth_head_wgrad(const void* x, const float* dy, float* dw, float* db, void* workspace,
                             size_t workspace_bytes, int n, int h, int wd, int c, void* stream) {
  if (!shape_ok(n, h, wd, c, "depth_head_wgrad")) return DIRB200_ERR_ARG;
  DIRB_CHECK_ARG(x && dy && dw && db && workspace, "depth_head_wgrad: null pointer");
  DIRB_CHECK_ARG(workspace_bytes >= wgrad_ws_bytes(n, h, wd, c),
                 "depth_head_wgrad: workspace too small (%zu bytes, needs %zu)", workspace_bytes,
                 wgrad_ws_bytes(n, h, wd, c));
  const int tiles = tiles_of(n, h, wd);
  float* part = static_cast<float*>(workspace);
  float* db_part = part + static_cast<size_t>(tiles) * 25 * c;
  depth_head_wgrad_partial_kernel<<<dim3(tiles, c / 8), WG_THREADS, 0, as_stream(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), dy, part, db_part, h, wd, c);
  DIRB_LAUNCHED();
  const int k_total = 25 * c;
  depth_head_wgrad_reduce_kernel<<<(k_total + 1 + 255) / 256, 256, 0, as_stream(stream)>>>(part, db_part, tiles, k_total,
                                                                                         dw, db);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
