// Dense-prediction ops of the NYUD2-DIR model around the convolutions (SURVEY §8f-2), NHWC bf16:
//   F.upsample(x, size, mode='bilinear')  (nyud2-dir/models/modules.py:24: align_corners = False)  forward + backward
//   torch.cat(..., 1)                      (modules.py:120: channel concat of the four MFF branches)  = a strided copy
// The convolutions themselves (5x5 / 3x3 / 1x1) are the wgmma implicit-GEMM kernels of conv_igemm.cu.
#include "common.cuh"

namespace dirb200 {

static inline int grid1d(int64_t n, int block = 256) {
  int64_t g = (n + block - 1) / block;
  const int64_t cap = 32 * static_cast<int64_t>(num_sms());
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

struct V8f { float v[8]; };
__device__ __forceinline__ V8f ld8(const __nv_bfloat16* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
  V8f r;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    r.v[2 * i] = f.x;
    r.v[2 * i + 1] = f.y;
  }
  return r;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const V8f& a) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a.v[2 * i], a.v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

// Bilinear up-sampling arithmetic, F.upsample(x, size, mode='bilinear') with align_corners = False
// (nyud2-dir/models/modules.py:24), as ATen forms it.  The fma contraction is written out: it is the one nvcc chose for
// the plain-C++ form of these lines (sm_90a, -O3), so no compiler setting can move the rounding.
//
// source index: s = max(scale * (dst + 0.5) - 0.5, 0), scale = in / out (float); i0 = floor(s) clamped to in - 1,
// i1 = min(i0 + 1, in - 1), lambda1 = s - i0
__device__ __forceinline__ void upsample_src_index(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
  float s = __fmaf_rn(__fadd_rn(static_cast<float>(dst), 0.5f), scale, -0.5f);
  if (s < 0.f) s = 0.f;
  i0 = static_cast<int>(s);
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = __fsub_rn(s, static_cast<float>(i0));
}

// ATen's association h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11), each sum an fma of its first product
// plus the rounded second product (hy = 1 - ly, hx = 1 - lx)
__device__ __forceinline__ float upsample_lerp(float v00, float v01, float v10, float v11, float hx, float lx, float hy,
                                               float ly) {
  const float top = __fmaf_rn(hx, v00, __fmul_rn(lx, v01));
  const float bot = __fmaf_rn(hx, v10, __fmul_rn(lx, v11));
  return __fmaf_rn(hy, top, __fmul_rn(ly, bot));
}

__global__ void __launch_bounds__(256)
upsample_bilinear_fwd_kernel(const __nv_bfloat16* __restrict__ x, int n, int h, int w, int c, int ho, int wo,
                             float sh, float sw, __nv_bfloat16* __restrict__ out) {
  const int cg = c / 8;
  const int64_t total = static_cast<int64_t>(n) * ho * wo * cg;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % cg);
    int64_t t = i / cg;
    const int ox = static_cast<int>(t % wo); t /= wo;
    const int oy = static_cast<int>(t % ho);
    const int b = static_cast<int>(t / ho);
    int y0, y1, x0, x1;
    float ly, lx;
    upsample_src_index(oy, sh, h, y0, y1, ly);
    upsample_src_index(ox, sw, w, x0, x1, lx);
    const __nv_bfloat16* base = x + static_cast<int64_t>(b) * h * w * c + g * 8;
    const V8f v00 = ld8(base + (static_cast<int64_t>(y0) * w + x0) * c), v01 = ld8(base + (static_cast<int64_t>(y0) * w + x1) * c);
    const V8f v10 = ld8(base + (static_cast<int64_t>(y1) * w + x0) * c), v11 = ld8(base + (static_cast<int64_t>(y1) * w + x1) * c);
    const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
    V8f o;
#pragma unroll
    for (int j = 0; j < 8; ++j) o.v[j] = upsample_lerp(v00.v[j], v01.v[j], v10.v[j], v11.v[j], hx, lx, hy, ly);
    st8(out + ((static_cast<int64_t>(b) * ho + oy) * wo + ox) * c + g * 8, o);
  }
}

// Backward as a GATHER (deterministic; ATen scatters with atomics): input pixel (iy, ix) collects w_y * w_x * dy from every
// output pixel whose two source rows / columns include it.  Candidate output rows are those with source position in
// (iy - 1, iy + 1): oy in [ (iy - 1 + 0.5) / sh - 0.5, (iy + 1 + 0.5) / sh - 0.5 ], widened by one and re-checked
// exactly with upsample_src_index.
__device__ __forceinline__ void candidates(int i, float scale, int out_size, int& lo, int& hi) {
  const float inv = 1.f / scale;
  lo = static_cast<int>(floorf((static_cast<float>(i) - 0.5f) * inv - 0.5f)) - 1;
  hi = static_cast<int>(ceilf((static_cast<float>(i) + 1.5f) * inv - 0.5f)) + 1;
  if (lo < 0) lo = 0;
  if (hi > out_size - 1) hi = out_size - 1;
}

__global__ void __launch_bounds__(256)
upsample_bilinear_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int n, int h, int w, int c, int ho, int wo, float sh,
                             float sw, __nv_bfloat16* __restrict__ dx) {
  const int cg = c / 8;
  const int64_t total = static_cast<int64_t>(n) * h * w * cg;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % cg);
    int64_t t = i / cg;
    const int ix = static_cast<int>(t % w); t /= w;
    const int iy = static_cast<int>(t % h);
    const int b = static_cast<int>(t / h);
    int ylo, yhi, xlo, xhi;
    candidates(iy, sh, ho, ylo, yhi);
    candidates(ix, sw, wo, xlo, xhi);
    V8f acc{};
    const __nv_bfloat16* base = dy + static_cast<int64_t>(b) * ho * wo * c + g * 8;
    for (int oy = ylo; oy <= yhi; ++oy) {
      int y0, y1;
      float ly;
      upsample_src_index(oy, sh, h, y0, y1, ly);
      const float wy = (y0 == iy ? 1.f - ly : 0.f) + (y1 == iy ? ly : 0.f);
      if (wy == 0.f) continue;
      for (int ox = xlo; ox <= xhi; ++ox) {
        int x0, x1;
        float lx;
        upsample_src_index(ox, sw, w, x0, x1, lx);
        const float wx = (x0 == ix ? 1.f - lx : 0.f) + (x1 == ix ? lx : 0.f);
        if (wx == 0.f) continue;
        const V8f gq = ld8(base + (static_cast<int64_t>(oy) * wo + ox) * c);
        const float wgt = wy * wx;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc.v[j] = fmaf(wgt, gq.v[j], acc.v[j]);
      }
    }
    st8(dx + ((static_cast<int64_t>(b) * h + iy) * w + ix) * c + g * 8, acc);
  }
}

// dst[p][dst_off + j] = src[p][src_off + j], j < c  (row strides in elements): channel concat / split of NHWC tensors
__global__ void __launch_bounds__(256)
copy_channels_kernel(const __nv_bfloat16* __restrict__ src, int src_stride, int src_off, __nv_bfloat16* __restrict__ dst,
                     int dst_stride, int dst_off, int c, int64_t pixels) {
  const int cg = c / 8;
  const int64_t total = pixels * cg;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % cg);
    const int64_t p = i / cg;
    *reinterpret_cast<uint4*>(dst + p * dst_stride + dst_off + g * 8) =
        *reinterpret_cast<const uint4*>(src + p * src_stride + src_off + g * 8);
  }
}

}  // namespace dirb200

using namespace dirb200;

extern "C" {

int dirb200_upsample_bilinear_fwd(const void* x, int n, int h, int w, int c, int ho, int wo, void* out, void* stream) {
  DIRB_CHECK_ARG(x && out && n > 0 && h > 0 && w > 0 && ho > 0 && wo > 0 && c > 0 && c % 8 == 0,
                 "upsample_bilinear_fwd: bad arguments (channels must be a multiple of 8)");
  upsample_bilinear_fwd_kernel<<<grid1d(static_cast<int64_t>(n) * ho * wo * (c / 8)), 256, 0, as_stream(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), n, h, w, c, ho, wo, static_cast<float>(h) / ho, static_cast<float>(w) / wo,
      static_cast<__nv_bfloat16*>(out));
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_upsample_bilinear_bwd(const void* dy, int n, int h, int w, int c, int ho, int wo, void* dx, void* stream) {
  DIRB_CHECK_ARG(dy && dx && n > 0 && h > 0 && w > 0 && ho > 0 && wo > 0 && c > 0 && c % 8 == 0,
                 "upsample_bilinear_bwd: bad arguments (channels must be a multiple of 8)");
  upsample_bilinear_bwd_kernel<<<grid1d(static_cast<int64_t>(n) * h * w * (c / 8)), 256, 0, as_stream(stream)>>>(
      static_cast<const __nv_bfloat16*>(dy), n, h, w, c, ho, wo, static_cast<float>(h) / ho, static_cast<float>(w) / wo,
      static_cast<__nv_bfloat16*>(dx));
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_copy_channels(const void* src, int src_stride, int src_off, void* dst, int dst_stride, int dst_off, int c,
                          int64_t pixels, void* stream) {
  DIRB_CHECK_ARG(src && dst && c > 0 && c % 8 == 0 && src_stride % 8 == 0 && dst_stride % 8 == 0 && src_off >= 0 &&
                     dst_off >= 0 && src_off % 8 == 0 && dst_off % 8 == 0 && src_off + c <= src_stride &&
                     dst_off + c <= dst_stride && pixels >= 0,
                 "copy_channels: channel counts / offsets / strides must be multiples of 8 and in range");
  if (pixels == 0) return DIRB200_OK;
  copy_channels_kernel<<<grid1d(pixels * (c / 8)), 256, 0, as_stream(stream)>>>(
      static_cast<const __nv_bfloat16*>(src), src_stride, src_off, static_cast<__nv_bfloat16*>(dst), dst_stride, dst_off, c,
      pixels);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
