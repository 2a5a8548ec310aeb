// HBM-bound layers of the ResNet stack around the wgmma convolutions, NHWC bf16:
// batch-norm (training statistics, apply(+residual)(+ReLU), backward), 3x3/2 max-pool,
// global average pool, the 2048->1 regressor and the fused Adam / SGD step.
// Replaces nn.BatchNorm2d / nn.ReLU / nn.MaxPool2d / nn.AvgPool2d / nn.Linear of
// agedb-dir/resnet.py:41-70,79-88,127-148 and torch.optim of agedb-dir/train.py:163-164.
#include "common.cuh"
#include "conv.cuh"
#include "nn.cuh"

namespace dirb200 {

constexpr int kReduceCtasPerSm = 4;   // grid cap of the column reductions (bounds the per-CTA partial buffer)

struct V8 {
  float v[8];
};
__device__ __forceinline__ V8 load8(const __nv_bfloat16* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
  V8 r;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    r.v[2 * i] = f.x;
    r.v[2 * i + 1] = f.y;
  }
  return r;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const V8& a) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a.v[2 * i], a.v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ V8 loadf8(const float* p) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  return V8{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}};
}

__device__ __forceinline__ float2 bf2_to_f2(uint32_t w) {
  return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}

// Column (per-channel) reduction over the rows of [P][C]: thread owns channel group cg = tid % (C/8) and walks
// rows with K partial sums per channel; the CTA combines its row-lanes in smem and writes ONE partial vector
// partial[blockIdx.x][k][c] (fp32, no atomics -> deterministic); the tiny per-channel finalize kernels add the
// partials of all CTAs in fp64.
template <int K>
__device__ __forceinline__ void column_reduce_finish(float (&acc)[K][8], int cg, int cgroups, int c,
                                                     float* __restrict__ partial) {
  extern __shared__ float sh[];  // [lanes][cgroups][K][8]
  const int lanes = blockDim.x / cgroups;
  float* mine = sh + threadIdx.x * (K * 8);      // threadIdx.x == lane * cgroups + cg
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) mine[k * 8 + j] = acc[k][j];
  __syncthreads();
  const int per_lane = cgroups * K * 8;           // == K * c
  float* out = partial + static_cast<size_t>(blockIdx.x) * K * c;
  for (int o = threadIdx.x; o < per_lane; o += blockDim.x) {
    float t = 0.f;
    for (int l = 0; l < lanes; ++l) t += sh[l * per_lane + o];
    const int g = o / (K * 8), k = (o / 8) % K, j = o & 7;
    out[k * c + g * 8 + j] = t;
  }
}

// Sums of two slots (s0, s1) of the per-CTA partials [nblocks][K][c] for channel ch, computed by a (32, 32) thread
// block: the 32 warps stride over the CTAs, 32 lanes cover 32 consecutive channels (coalesced 128-byte reads), and
// both slots are fetched in the same pass so that four independent loads are in flight per thread (these tiny
// kernels sit on the critical path between two streaming kernels, 106 times per step: pure latency).
// Valid in threads with threadIdx.y == 0 after the call.
__device__ __forceinline__ void sum_partials2(const float* __restrict__ partial, int nblocks, int K, int s0, int s1,
                                              int c, int ch, double (*sh)[32], double& r0, double& r1) {
  double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
  if (ch < c) {
    int b = threadIdx.y;
    for (; b + 32 < nblocks; b += 64) {
      const float x0 = partial[((size_t)b * K + s0) * c + ch];
      const float y0 = partial[((size_t)b * K + s1) * c + ch];
      const float x1 = partial[((size_t)(b + 32) * K + s0) * c + ch];
      const float y1 = partial[((size_t)(b + 32) * K + s1) * c + ch];
      a0 += (double)x0;
      b0 += (double)y0;
      a1 += (double)x1;
      b1 += (double)y1;
    }
    if (b < nblocks) {
      a0 += (double)partial[((size_t)b * K + s0) * c + ch];
      b0 += (double)partial[((size_t)b * K + s1) * c + ch];
    }
  }
  sh[threadIdx.y][threadIdx.x] = a0 + a1;
  __syncthreads();
  r0 = 0.0;
  if (threadIdx.y == 0)
    for (int w = 0; w < 32; ++w) r0 += sh[w][threadIdx.x];
  __syncthreads();
  sh[threadIdx.y][threadIdx.x] = b0 + b1;
  __syncthreads();
  r1 = 0.0;
  if (threadIdx.y == 0)
    for (int w = 0; w < 32; ++w) r1 += sh[w][threadIdx.x];
  __syncthreads();
}

__global__ void __launch_bounds__(256, 4)
bn_stats_kernel(const __nv_bfloat16* __restrict__ y, int64_t rows, int c, float* __restrict__ partial) {
  const int cgroups = c / 8;
  const int cg = threadIdx.x % cgroups, lane = threadIdx.x / cgroups, lanes = blockDim.x / cgroups;
  float acc[2][8] = {};
  const int64_t stride = (int64_t)gridDim.x * lanes;
  int64_t r = blockIdx.x * (int64_t)lanes + lane;
  // 4 independent 16-byte loads in flight per thread
  for (; r + 3 * stride < rows; r += 4 * stride) {
    V8 x[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) x[u] = load8(y + (r + u * stride) * c + cg * 8);
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[0][j] += x[u].v[j];
        acc[1][j] = fmaf(x[u].v[j], x[u].v[j], acc[1][j]);
      }
  }
  for (; r < rows; r += stride) {
    const V8 x = load8(y + r * c + cg * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[0][j] += x.v[j];
      acc[1][j] = fmaf(x.v[j], x.v[j], acc[1][j]);
    }
  }
  column_reduce_finish<2>(acc, cg, cgroups, c, partial);
}

// Sums of the two slots of the per-CTA rows [rows][2][c] that hold channel i under layout L (conv epilogue statistics,
// see StatLayout): CTA groups j, j + n_tiles, ...; `group` consecutive rows each.  (32, 32) thread block as above;
// valid in threads with threadIdx.y == 0 after the call.
__device__ __forceinline__ void sum_layout2(const float* __restrict__ partial, const StatLayout& L, int c, int i,
                                            double (*sh)[32][32], double& r0, double& r1) {
  double a0 = 0.0, b0 = 0.0, a1 = 0.0, b1 = 0.0;
  if (i < c) {
    const int j = i / L.bn;
    const int ngroups = L.rows / L.group;
    const int nk = j < ngroups ? (ngroups - 1 - j) / L.n_tiles + 1 : 0;
    const int nrows = nk * L.group;
    int t = threadIdx.y;
    for (; t + 32 < nrows; t += 64) {            // four independent loads in flight
      const int q0 = (j + (t / L.group) * L.n_tiles) * L.group + t % L.group;
      const int q1 = (j + ((t + 32) / L.group) * L.n_tiles) * L.group + (t + 32) % L.group;
      const float x0 = partial[((size_t)q0 * 2) * c + i], y0 = partial[((size_t)q0 * 2 + 1) * c + i];
      const float x1 = partial[((size_t)q1 * 2) * c + i], y1 = partial[((size_t)q1 * 2 + 1) * c + i];
      a0 += (double)x0; b0 += (double)y0; a1 += (double)x1; b1 += (double)y1;
    }
    if (t < nrows) {
      const int q0 = (j + (t / L.group) * L.n_tiles) * L.group + t % L.group;
      a0 += (double)partial[((size_t)q0 * 2) * c + i];
      b0 += (double)partial[((size_t)q0 * 2 + 1) * c + i];
    }
  }
  sh[0][threadIdx.y][threadIdx.x] = a0 + a1;
  sh[1][threadIdx.y][threadIdx.x] = b0 + b1;
  __syncthreads();
  r0 = r1 = 0.0;
  if (threadIdx.y == 0)
    for (int w = 0; w < 32; ++w) {
      r0 += sh[0][w][threadIdx.x];
      r1 += sh[1][w][threadIdx.x];
    }
}

// mean / invstd / scale / shift from the accumulated sums; running statistics as nn.BatchNorm2d (momentum 0.1,
// unbiased running variance).
__global__ void bn_finalize_kernel(const float* __restrict__ partial, StatLayout L, int64_t rows, int c,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float momentum, float* __restrict__ running_mean, float* __restrict__ running_var,
                                   float* __restrict__ mean_out, float* __restrict__ invstd_out,
                                   float* __restrict__ scale, float* __restrict__ shift) {
  __shared__ double sh[2][32][32];
  const int i = blockIdx.x * 32 + threadIdx.x;
  double sx, sq;
  sum_layout2(partial, L, c, i, sh, sx, sq);
  if (threadIdx.y != 0 || i >= c) return;
  const double n = (double)rows;
  const double m = sx / n;
  double var = sq / n - m * m;
  if (var < 0.0) var = 0.0;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  mean_out[i] = (float)m;
  invstd_out[i] = invstd;
  const float sc = gamma[i] * invstd;
  scale[i] = sc;
  shift[i] = beta[i] - (float)m * sc;
  if (running_mean) {
    const double unbiased = rows > 1 ? var * n / (n - 1.0) : var;
    running_mean[i] = (1.f - momentum) * running_mean[i] + momentum * (float)m;
    running_var[i] = (1.f - momentum) * running_var[i] + momentum * (float)unbiased;
  }
}

// eval mode: scale/shift from the running statistics
__global__ void bn_eval_coeffs_kernel(int c, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                      const float* __restrict__ running_mean, const float* __restrict__ running_var,
                                      float* __restrict__ scale, float* __restrict__ shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c) return;
  const float sc = gamma[i] * rsqrtf(running_var[i] + eps);
  scale[i] = sc;
  shift[i] = beta[i] - running_mean[i] * sc;
}

__global__ void bn_eval_coeffs_all_kernel(const BnEvalDesc* __restrict__ descs, const float* __restrict__ params,
                                          const float* __restrict__ running, float eps) {
  const BnEvalDesc d = descs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.c) return;
  const float sc = params[d.gamma_off + i] * rsqrtf(running[d.rv_off + i] + eps);
  d.scale[i] = sc;
  d.shift[i] = params[d.beta_off + i] - running[d.rm_off + i] * sc;
}

// out = [relu]( y*scale + shift  [+ res]  [+ res_y*res_scale + res_shift] )
// Thread = (channel group of 8, row lane): the per-channel coefficients are loaded once into registers and the
// thread walks rows (same mapping as the column reductions), so the streaming loop is pure 16-byte loads + FMAs.
__device__ __forceinline__ uint32_t f2_to_bf2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// mask_out (block outputs only): one byte per (row, channel group): bit j = out[row][cg*8 + j] > 0 -- the ReLU mask
// the backward kernels need, 1/16 of the size of `out`.
// Rows per iteration R (4 for the plain form, 2 with a residual): every load of all R rows is issued before the first
// use, so that several 16-byte loads per thread are in flight to cover the HBM latency (R has not been re-tuned on H100).
template <bool HAS_RES, bool HAS_RESY, bool MASK>
__global__ void __launch_bounds__(256)
bn_apply_kernel(const __nv_bfloat16* __restrict__ y, const float* __restrict__ scale, const float* __restrict__ shift,
                const __nv_bfloat16* __restrict__ res, const __nv_bfloat16* __restrict__ res_y,
                const float* __restrict__ res_scale, const float* __restrict__ res_shift, int relu, int64_t rows,
                int c, __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ mask_out) {
  constexpr int R = (HAS_RES || HAS_RESY) ? 2 : 4;
  const int cgroups = c / 8;
  const int cg = threadIdx.x % cgroups, lane = threadIdx.x / cgroups, lanes = blockDim.x / cgroups;
  const V8 sc = loadf8(scale + cg * 8), sh = loadf8(shift + cg * 8);
  V8 rs{}, rh{};
  if (HAS_RESY) {
    rs = loadf8(res_scale + cg * 8);
    rh = loadf8(res_shift + cg * 8);
  }
  const int64_t stride = (int64_t)gridDim.x * lanes;
  for (int64_t r0 = blockIdx.x * (int64_t)lanes + lane; r0 < rows; r0 += R * stride) {
    int64_t offs[R], rr[R];
    bool live[R];
    uint4 Y[R], RV[R];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      rr[u] = r0 + u * stride;
      live[u] = rr[u] < rows;
      if (!live[u]) rr[u] = r0;
      offs[u] = rr[u] * c + cg * 8;
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      Y[u] = *reinterpret_cast<const uint4*>(y + offs[u]);
      if (HAS_RES) RV[u] = *reinterpret_cast<const uint4*>(res + offs[u]);
      if (HAS_RESY) RV[u] = *reinterpret_cast<const uint4*>(res_y + offs[u]);
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      if (!live[u]) continue;
      const uint32_t yw[4] = {Y[u].x, Y[u].y, Y[u].z, Y[u].w}, rw[4] = {RV[u].x, RV[u].y, RV[u].z, RV[u].w};
      uint32_t ow[4];
      uint32_t bits = 0;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float2 yv = bf2_to_f2(yw[w]);
        float a = fmaf(yv.x, sc.v[2 * w], sh.v[2 * w]), b = fmaf(yv.y, sc.v[2 * w + 1], sh.v[2 * w + 1]);
        if (HAS_RES) {
          const float2 t = bf2_to_f2(rw[w]);
          a += t.x;
          b += t.y;
        }
        if (HAS_RESY) {
          const float2 t = bf2_to_f2(rw[w]);
          a += fmaf(t.x, rs.v[2 * w], rh.v[2 * w]);
          b += fmaf(t.y, rs.v[2 * w + 1], rh.v[2 * w + 1]);
        }
        if (relu) {
          a = fmaxf(a, 0.f);
          b = fmaxf(b, 0.f);
        }
        ow[w] = f2_to_bf2(a, b);
        // the stored (bf16-rounded) value > 0  <=>  magnitude bits non-zero after the ReLU
        bits |= ((ow[w] & 0x00007fffu) ? 1u : 0u) << (2 * w);
        bits |= ((ow[w] & 0x7fff0000u) ? 1u : 0u) << (2 * w + 1);
      }
      *reinterpret_cast<uint4*>(out + offs[u]) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      if (MASK) mask_out[rr[u] * cgroups + cg] = static_cast<uint8_t>(bits);
    }
  }
}

// ---- backward.  dz = (g1 [+ g2]) * relu_mask.  The mask is never read from an activation tensor:
//   MASK_FROM_Y  (conv -> BN -> ReLU):       mask = (y*scale + shift > 0), the same fmaf the forward evaluated, so the
//                                            activation `a` is not touched by the backward pass at all;
//   MASK_BITS    (block output, BN + residual + ReLU):  the 1-bit-per-element mask bn_apply stored.
// The reduction accumulates the raw moments  S0 = sum dz,  S1 = sum dz*y  [, S2 = sum dz*y2 for the downsample-branch
// BN that shares dz]; dbeta = S0 and dgamma = invstd * (S1 - mean*S0) are formed in fp64 by bn_bwd_coeffs_kernel.
enum { MASK_FROM_Y = 0, MASK_BITS = 1, MASK_NONE = 2 };   // MASK_NONE: the incoming tensor is dz already

template <int MODE>
struct MaskSrc {
  V8 sc, sh;                 // MASK_FROM_Y
  const uint8_t* bits;       // MASK_BITS
  int cgroups, cg;
  __device__ __forceinline__ void init(const float* scale, const float* shift, const uint8_t* b, int cgroups_, int cg_) {
    cgroups = cgroups_;
    cg = cg_;
    bits = b;
    if (MODE == MASK_FROM_Y) {
      sc = loadf8(scale + cg * 8);
      sh = loadf8(shift + cg * 8);
    }
  }
  __device__ __forceinline__ uint32_t load(int64_t r) const { return MODE == MASK_BITS ? bits[r * cgroups + cg] : 0u; }
  // keep-mask of channel pair w given the raw conv output pair yv
  __device__ __forceinline__ void apply(uint32_t m, int w, const float2& yv, float2& g) const {
    if (MODE == MASK_FROM_Y) {
      if (!(fmaf(yv.x, sc.v[2 * w], sh.v[2 * w]) > 0.f)) g.x = 0.f;
      if (!(fmaf(yv.y, sc.v[2 * w + 1], sh.v[2 * w + 1]) > 0.f)) g.y = 0.f;
    } else if (MODE == MASK_BITS) {
      if (!((m >> (2 * w)) & 1u)) g.x = 0.f;
      if (!((m >> (2 * w + 1)) & 1u)) g.y = 0.f;
    }
  }
};

// Second incoming gradient of a block output: absent, a dense tensor, or -- behind a stride-2 1x1 downsample conv --
// the COMPACT tensor [n, h/2, w/2, c] of that conv's dgrad, which contributes only at even (y, x) (the dense form
// would be a memset of the full map plus a scattered GEMM plus two dense re-reads of mostly zeros).
enum { G2_NONE = 0, G2_DENSE = 1, G2_COMPACT = 2 };
struct CompactG2 {
  FastDiv hw, w;          // full-resolution pixel grid of the rows
  int h2, w2;             // compact grid
  __device__ __forceinline__ bool locate(int64_t r, int64_t& r2) const {
    uint32_t n, rem, yy, xx;
    hw.divmod(static_cast<uint32_t>(r), n, rem);
    w.divmod(rem, yy, xx);
    r2 = (static_cast<int64_t>(n) * h2 + (yy >> 1)) * w2 + (xx >> 1);
    return ((yy | xx) & 1u) == 0u;
  }
};

// WRITE_DZ (identity blocks): dz is stored (bf16) -- it is the gradient of the shortcut path anyway -- and the sums
// are taken over the STORED values, so that bn_bwd_apply can read dz (one tensor) instead of g1, g2 and the mask again.
// HAS_G3 (identity blocks whose output is also a block output of the multi-scale encoder): a third dense gradient g3,
// added in fp32 to g1 + g2 before the mask and the one bf16 rounding of dz.
template <int MODE, int G2M, bool HAS_Y2, bool WRITE_DZ, bool HAS_G3 = false>
__global__ void __launch_bounds__(256, 3)
bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ g1, const __nv_bfloat16* __restrict__ g2, CompactG2 cg2,
                     const __nv_bfloat16* __restrict__ g3, const __nv_bfloat16* __restrict__ y,
                     const __nv_bfloat16* __restrict__ y2,
                     const float* __restrict__ scale, const float* __restrict__ shift,
                     const uint8_t* __restrict__ mask, int64_t rows, int c, float* __restrict__ partial,
                     __nv_bfloat16* __restrict__ dz_out) {
  constexpr bool HAS_G2 = G2M != G2_NONE;
  const int cgroups = c / 8;
  const int cg = threadIdx.x % cgroups, lane = threadIdx.x / cgroups, lanes = blockDim.x / cgroups;
  constexpr int K = HAS_Y2 ? 3 : 2;
  float acc[K][8] = {};
  MaskSrc<MODE> ms;
  ms.init(scale, shift, mask, cgroups, cg);
  const int64_t stride = (int64_t)gridDim.x * lanes;
  // two rows per iteration: every load of both rows is issued before the first use
  for (int64_t r0 = blockIdx.x * (int64_t)lanes + lane; r0 < rows; r0 += 2 * stride) {
    const int64_t r1 = r0 + stride;
    const bool two = r1 < rows;
    const int64_t o0 = r0 * c + cg * 8, o1 = (two ? r1 : r0) * c + cg * 8;
    uint4 G[2], Y[2], G2[2], Y2[2], G3[2];
    uint32_t M[2];
    G[0] = *reinterpret_cast<const uint4*>(g1 + o0);
    G[1] = *reinterpret_cast<const uint4*>(g1 + o1);
    if (HAS_G3) {
      G3[0] = *reinterpret_cast<const uint4*>(g3 + o0);
      G3[1] = *reinterpret_cast<const uint4*>(g3 + o1);
    }
    Y[0] = *reinterpret_cast<const uint4*>(y + o0);
    Y[1] = *reinterpret_cast<const uint4*>(y + o1);
    if (G2M == G2_DENSE) {
      G2[0] = *reinterpret_cast<const uint4*>(g2 + o0);
      G2[1] = *reinterpret_cast<const uint4*>(g2 + o1);
    } else if (G2M == G2_COMPACT) {
      int64_t q0, q1;
      const bool v0 = cg2.locate(r0, q0), v1 = cg2.locate(two ? r1 : r0, q1);
      G2[0] = v0 ? *reinterpret_cast<const uint4*>(g2 + q0 * c + cg * 8) : make_uint4(0, 0, 0, 0);
      G2[1] = v1 ? *reinterpret_cast<const uint4*>(g2 + q1 * c + cg * 8) : make_uint4(0, 0, 0, 0);
    }
    if (HAS_Y2) {
      Y2[0] = *reinterpret_cast<const uint4*>(y2 + o0);
      Y2[1] = *reinterpret_cast<const uint4*>(y2 + o1);
    }
    M[0] = ms.load(r0);
    M[1] = ms.load(two ? r1 : r0);
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (u == 1 && !two) break;
      const uint32_t gw[4] = {G[u].x, G[u].y, G[u].z, G[u].w}, yw[4] = {Y[u].x, Y[u].y, Y[u].z, Y[u].w};
      uint32_t oz[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        float2 g = bf2_to_f2(gw[w]);
        if (HAS_G2) {
          const uint32_t g2w[4] = {G2[u].x, G2[u].y, G2[u].z, G2[u].w};
          const float2 t = bf2_to_f2(g2w[w]);
          g.x += t.x;
          g.y += t.y;
        }
        if (HAS_G3) {
          const uint32_t g3w[4] = {G3[u].x, G3[u].y, G3[u].z, G3[u].w};
          const float2 t = bf2_to_f2(g3w[w]);
          g.x += t.x;
          g.y += t.y;
        }
        const float2 yv = bf2_to_f2(yw[w]);
        ms.apply(M[u], w, yv, g);
        if (WRITE_DZ) {
          oz[w] = f2_to_bf2(g.x, g.y);
          g = bf2_to_f2(oz[w]);
        }
        acc[0][2 * w] += g.x;
        acc[0][2 * w + 1] += g.y;
        acc[1][2 * w] = fmaf(g.x, yv.x, acc[1][2 * w]);
        acc[1][2 * w + 1] = fmaf(g.y, yv.y, acc[1][2 * w + 1]);
        if (HAS_Y2) {
          const uint32_t y2w[4] = {Y2[u].x, Y2[u].y, Y2[u].z, Y2[u].w};
          const float2 y2v = bf2_to_f2(y2w[w]);
          acc[K - 1][2 * w] = fmaf(g.x, y2v.x, acc[K - 1][2 * w]);
          acc[K - 1][2 * w + 1] = fmaf(g.y, y2v.y, acc[K - 1][2 * w + 1]);
        }
      }
      if (WRITE_DZ) *reinterpret_cast<uint4*>(dz_out + (u ? o1 : o0)) = make_uint4(oz[0], oz[1], oz[2], oz[3]);
    }
  }
  column_reduce_finish<K>(acc, cg, cgroups, c, partial);
}

// Per-channel coefficients of the BN backward, dy = A*dz + B*y + C with
//   A = gamma*invstd,  B = -gamma*invstd^2*dgamma/n,  C = gamma*invstd*(mean*invstd*dgamma/n - dbeta/n);
// dbeta / dgamma are summed here from the reduce kernel's per-CTA partials [nblocks][K][c] (dbeta = slot 0,
// dgamma = slot `gslot`); also accumulates them into the fp32 parameter gradients.
__device__ __forceinline__ void bn_bwd_coeffs_write(double db, double s1, int i, int64_t rows, int c,
                                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                                    const float* __restrict__ gamma, float* __restrict__ grad_gamma,
                                                    float* __restrict__ grad_beta, float* __restrict__ coef) {
  const double n = (double)rows, is = (double)invstd[i], ga = (double)gamma[i], mu = (double)mean[i];
  const double dg = is * (s1 - mu * db);          // sum dz * xhat from the raw moments
  coef[i] = (float)(ga * is);
  coef[c + i] = (float)(-ga * is * is * dg / n);
  coef[2 * c + i] = (float)(ga * is * (mu * is * dg / n - db / n));
  grad_gamma[i] += (float)dg;
  grad_beta[i] += (float)db;
}

__global__ void bn_bwd_coeffs_kernel(const float* __restrict__ partial, int nblocks, int K, int gslot, int64_t rows,
                                     int c, const float* __restrict__ mean, const float* __restrict__ invstd,
                                     const float* __restrict__ gamma, float* __restrict__ grad_gamma,
                                     float* __restrict__ grad_beta, float* __restrict__ coef /* [3][c] */) {
  __shared__ double sh[32][32];
  const int i = blockIdx.x * 32 + threadIdx.x;
  double db, s1;
  sum_partials2(partial, nblocks, K, 0, gslot, c, i, sh, db, s1);
  if (threadIdx.y != 0 || i >= c) return;
  bn_bwd_coeffs_write(db, s1, i, rows, c, mean, invstd, gamma, grad_gamma, grad_beta, coef);
}

// same, from the per-CTA rows a dgrad epilogue wrote (conv_dgrad with DgradBnMoments; rows as L describes)
__global__ void bn_bwd_coeffs_layout_kernel(const float* __restrict__ partial, StatLayout L, int64_t rows, int c,
                                            const float* __restrict__ mean, const float* __restrict__ invstd,
                                            const float* __restrict__ gamma, float* __restrict__ grad_gamma,
                                            float* __restrict__ grad_beta, float* __restrict__ coef) {
  __shared__ double sh[2][32][32];
  const int i = blockIdx.x * 32 + threadIdx.x;
  double db, s1;
  sum_layout2(partial, L, c, i, sh, db, s1);
  if (threadIdx.y != 0 || i >= c) return;
  bn_bwd_coeffs_write(db, s1, i, rows, c, mean, invstd, gamma, grad_gamma, grad_beta, coef);
}

// dz = (g1 [+ g2]) * mask;  dy = A*dz + B*y + C  (and the same for the second BN);  optionally writes dz.
// Same (channel group, row lane) mapping as bn_apply: coefficients live in registers.
template <int MODE, int G2M, bool HAS_Y2, bool WRITE_DZ>
__global__ void __launch_bounds__(256, 2)
bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ g1, const __nv_bfloat16* __restrict__ g2, CompactG2 cg2,
                    const __nv_bfloat16* __restrict__ y, const float* __restrict__ coef,
                    const __nv_bfloat16* __restrict__ y2, const float* __restrict__ coef2,
                    const float* __restrict__ scale, const float* __restrict__ shift,
                    const uint8_t* __restrict__ mask, int64_t rows, int c, __nv_bfloat16* __restrict__ dy,
                    __nv_bfloat16* __restrict__ dy2, __nv_bfloat16* __restrict__ dz_out) {
  // rows per iteration: every load of all of them is issued before the first use.  Two CTAs of 8 warps fit per SM
  // (register-limited), so the plain two-input form keeps four rows (8 x 16 B per thread) in flight to cover the HBM
  // latency; the forms with more inputs keep two (not re-tuned on H100).
  constexpr bool HAS_G2 = G2M != G2_NONE;
  constexpr int R = (HAS_G2 || HAS_Y2) ? 2 : 4;
  const int cgroups = c / 8;
  const int cg = threadIdx.x % cgroups, lane = threadIdx.x / cgroups, lanes = blockDim.x / cgroups;
  const V8 A = loadf8(coef + cg * 8), B = loadf8(coef + c + cg * 8), C = loadf8(coef + 2 * c + cg * 8);
  V8 A2{}, B2{}, C2{};
  if (HAS_Y2) {
    A2 = loadf8(coef2 + cg * 8);
    B2 = loadf8(coef2 + c + cg * 8);
    C2 = loadf8(coef2 + 2 * c + cg * 8);
  }
  MaskSrc<MODE> ms;
  ms.init(scale, shift, mask, cgroups, cg);
  const int64_t stride = (int64_t)gridDim.x * lanes;
  for (int64_t r0 = blockIdx.x * (int64_t)lanes + lane; r0 < rows; r0 += R * stride) {
    int64_t rr[R], offs[R];
    bool live[R];
    uint4 G[R], Y[R], G2[R], Y2[R];
    uint32_t M[R];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      rr[u] = r0 + u * stride;
      live[u] = rr[u] < rows;
      if (!live[u]) rr[u] = r0;
      offs[u] = rr[u] * c + cg * 8;
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      G[u] = *reinterpret_cast<const uint4*>(g1 + offs[u]);
      Y[u] = *reinterpret_cast<const uint4*>(y + offs[u]);
      if (G2M == G2_DENSE) {
        G2[u] = *reinterpret_cast<const uint4*>(g2 + offs[u]);
      } else if (G2M == G2_COMPACT) {
        int64_t q;
        const bool v = cg2.locate(rr[u], q);
        G2[u] = v ? *reinterpret_cast<const uint4*>(g2 + q * c + cg * 8) : make_uint4(0, 0, 0, 0);
      }
      if (HAS_Y2) Y2[u] = *reinterpret_cast<const uint4*>(y2 + offs[u]);
      M[u] = ms.load(rr[u]);
    }
#pragma unroll
    for (int u = 0; u < R; ++u) {
      if (!live[u]) continue;
      const uint32_t gw[4] = {G[u].x, G[u].y, G[u].z, G[u].w}, yw[4] = {Y[u].x, Y[u].y, Y[u].z, Y[u].w};
      uint32_t o1[4], o2[4], oz[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        float2 g = bf2_to_f2(gw[w]);
        if (HAS_G2) {
          const uint32_t g2w[4] = {G2[u].x, G2[u].y, G2[u].z, G2[u].w};
          const float2 t = bf2_to_f2(g2w[w]);
          g.x += t.x;
          g.y += t.y;
        }
        const float2 yv = bf2_to_f2(yw[w]);
        ms.apply(M[u], w, yv, g);
        if (WRITE_DZ) oz[w] = f2_to_bf2(g.x, g.y);
        o1[w] = f2_to_bf2(fmaf(A.v[2 * w], g.x, fmaf(B.v[2 * w], yv.x, C.v[2 * w])),
                          fmaf(A.v[2 * w + 1], g.y, fmaf(B.v[2 * w + 1], yv.y, C.v[2 * w + 1])));
        if (HAS_Y2) {
          const uint32_t y2w[4] = {Y2[u].x, Y2[u].y, Y2[u].z, Y2[u].w};
          const float2 y2v = bf2_to_f2(y2w[w]);
          o2[w] = f2_to_bf2(fmaf(A2.v[2 * w], g.x, fmaf(B2.v[2 * w], y2v.x, C2.v[2 * w])),
                            fmaf(A2.v[2 * w + 1], g.y, fmaf(B2.v[2 * w + 1], y2v.y, C2.v[2 * w + 1])));
        }
      }
      *reinterpret_cast<uint4*>(dy + offs[u]) = make_uint4(o1[0], o1[1], o1[2], o1[3]);
      if (HAS_Y2) *reinterpret_cast<uint4*>(dy2 + offs[u]) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
      if (WRITE_DZ) *reinterpret_cast<uint4*>(dz_out + offs[u]) = make_uint4(oz[0], oz[1], oz[2], oz[3]);
    }
  }
}

// ------------------------------------------------------------------ pooling
// 3x3 / stride 2 / pad 1 max pool; idx = r*3+s of the first maximum (PyTorch's tie rule)
__global__ void maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, int n, int h, int w, int c,
                                   __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ idx) {
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1, cg = c / 8;
  const int64_t total = (int64_t)n * ho * wo * cg;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    int64_t t = i / cg;
    const int xo = (int)(t % wo); t /= wo;
    const int yo = (int)(t % ho);
    const int b = (int)(t / ho);
    float best[8];
    int bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; bi[j] = 0; }
    for (int r = 0; r < 3; ++r) {
      const int yi = 2 * yo - 1 + r;
      if (yi < 0 || yi >= h) continue;
      for (int s = 0; s < 3; ++s) {
        const int xi = 2 * xo - 1 + s;
        if (xi < 0 || xi >= w) continue;
        const V8 v = load8(x + (((int64_t)b * h + yi) * w + xi) * c + g * 8);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (v.v[j] > best[j]) { best[j] = v.v[j]; bi[j] = r * 3 + s; }
      }
    }
    V8 o;
    __align__(8) uint8_t ib[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { o.v[j] = best[j]; ib[j] = (uint8_t)bi[j]; }
    const int64_t off = (((int64_t)b * ho + yo) * wo + xo) * c + g * 8;
    store8(out + off, o);
    *reinterpret_cast<uint2*>(idx + off) = *reinterpret_cast<uint2*>(ib);
  }
}

// Stem: relu(bn(y)) and the 3x3 / stride 2 / pad 1 max pool in one pass (resnet.py:128-131: bn1 -> relu -> maxpool).
// The activation is never written: the backward re-derives the ReLU mask from (y, scale, shift) and routes gradients by
// the stored argmax, so nothing downstream reads it (saves 411 MB written + read at batch 256).  Values are rounded to
// bf16 before they are compared, i.e. exactly what pooling the stored activation gave; idx = r*3+s of the first maximum.
// A thread owns a 2x2 block of OUTPUT pixels x 8 channels: the 5x5 input patch they cover is loaded once (6.25 loads and
// BN+ReLU evaluations per output instead of 9) row by row -- five 16-byte loads in flight.  Running maximum AND argmax
// of a window live in ONE integer per channel: key = (bf16 bits of the activation << 4) | (15 - pos).  Activations are
// >= 0 after the ReLU, so their bf16 bit patterns order like the values, and on equal values the smaller filter position
// wins (PyTorch's first-maximum rule); an update is one OR + one integer max instead of a compare, a select and a
// byte insert (the kernel was ALU-bound on those).
__global__ void __launch_bounds__(256)
bn_relu_maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ y, const float* __restrict__ scale,
                           const float* __restrict__ shift, int n, int h, int w, int c,
                           __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ idx) {
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1, cg = c / 8;
  const int hb = (ho + 1) / 2, wb = (wo + 1) / 2;
  const int64_t total = (int64_t)n * hb * wb * cg;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    int64_t t = i / cg;
    const int xb = (int)(t % wb); t /= wb;
    const int yb = (int)(t % hb);
    const int b = (int)(t / hb);
    const V8 sc = loadf8(scale + g * 8), sh = loadf8(shift + g * 8);
    uint32_t best[4][8];                 // [oy * 2 + ox][channel]: (bf16 bits << 4) | (15 - pos)
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) best[k][j] = 0u;
    const int y0 = 4 * yb - 1, x0 = 4 * xb - 1;     // first input row / column of the 5x5 patch
#pragma unroll
    for (int ry = 0; ry < 5; ++ry) {
      const int yi = y0 + ry;
      const bool yok = yi >= 0 && yi < h;
      uint4 v[5];
#pragma unroll
      for (int cx = 0; cx < 5; ++cx) {
        const int xi = x0 + cx;
        v[cx] = (yok && xi >= 0 && xi < w) ? *reinterpret_cast<const uint4*>(y + (((int64_t)b * h + yi) * w + xi) * c + g * 8)
                                           : make_uint4(0, 0, 0, 0);
      }
      if (!yok) continue;
#pragma unroll
      for (int cx = 0; cx < 5; ++cx) {
        const int xi = x0 + cx;
        if (xi < 0 || xi >= w) continue;
        const uint32_t yw[4] = {v[cx].x, v[cx].y, v[cx].z, v[cx].w};
        uint32_t kb[8];                  // bf16 bits of relu(bn(y)) << 4
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float2 yv = bf2_to_f2(yw[p]);
          const uint32_t pk = f2_to_bf2(fmaxf(fmaf(yv.x, sc.v[2 * p], sh.v[2 * p]), 0.f),
                                        fmaxf(fmaf(yv.y, sc.v[2 * p + 1], sh.v[2 * p + 1]), 0.f));
          kb[2 * p] = (pk & 0x7fffu) << 4;                  // (sign bit dropped: a ReLU output of -0 counts as 0)
          kb[2 * p + 1] = (pk >> 12) & 0x7fff0u;
        }
#pragma unroll
        for (int oy = 0; oy < 2; ++oy) {
          const int r = ry - 2 * oy;                 // filter row of this input row in output row oy
          if (r < 0 || r > 2) continue;
#pragma unroll
          for (int ox = 0; ox < 2; ++ox) {
            const int q = cx - 2 * ox;
            if (q < 0 || q > 2) continue;
            const uint32_t tie = 15u - (uint32_t)(r * 3 + q);
            const int k = oy * 2 + ox;
#pragma unroll
            for (int j = 0; j < 8; ++j) best[k][j] = max(best[k][j], kb[j] | tie);
          }
        }
      }
    }
#pragma unroll
    for (int oy = 0; oy < 2; ++oy)
#pragma unroll
      for (int ox = 0; ox < 2; ++ox) {
        const int yo = 2 * yb + oy, xo = 2 * xb + ox;
        if (yo >= ho || xo >= wo) continue;
        const uint32_t* bk = best[oy * 2 + ox];
        uint32_t ow[4], iw[2] = {0u, 0u};
#pragma unroll
        for (int p = 0; p < 4; ++p) ow[p] = (bk[2 * p] >> 4) | ((bk[2 * p + 1] >> 4) << 16);
#pragma unroll
        for (int j = 0; j < 8; ++j) iw[j >> 2] |= (15u - (bk[j] & 15u)) << (8 * (j & 3));
        const int64_t off = (((int64_t)b * ho + yo) * wo + xo) * c + g * 8;
        *reinterpret_cast<uint4*>(out + off) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        *reinterpret_cast<uint2*>(idx + off) = make_uint2(iw[0], iw[1]);
      }
  }
}

// dx[h,w] = sum over the (<= 4) windows containing (h,w) whose argmax is this position of (g1 [+ g2]).
// A thread owns a 2x2 block of input pixels (2a+py, 2b+px) x 8 channels: exactly the four windows (a+dy, b+dx) reach
// it, so each window's (gradient, argmax) is loaded once per block instead of once per covered pixel (2.25 loads per
// pixel on average before) and all four loads are issued before any is consumed.  Pixel (py, px) sits at filter
// position ((py + 1 - 2 dy), (px + 1 - 2 dx)) of window (dy, dx) -- inside the 3x3 only if (dy == 0 || py == 1) and
// (dx == 0 || px == 1).  H, W even (the runner's stem output always is).
__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ g1, const __nv_bfloat16* __restrict__ g2,
                   const uint8_t* __restrict__ idx, int n, int h, int w, int c, __nv_bfloat16* __restrict__ dx) {
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1, cg = c / 8;
  const int hb = h / 2, wb = w / 2;
  const int64_t total = (int64_t)n * hb * wb * cg;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    int64_t t = i / cg;
    const int xb = (int)(t % wb); t /= wb;
    const int ya = (int)(t % hb);
    const int b = (int)(t / hb);
    uint4 gv[4], g2v[4];
    uint2 iv[4];
    bool ok[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yo = ya + (k >> 1), xo = xb + (k & 1);
      ok[k] = yo < ho && xo < wo;
      const int64_t off = (((int64_t)b * ho + (ok[k] ? yo : 0)) * wo + (ok[k] ? xo : 0)) * c + g * 8;
      gv[k] = *reinterpret_cast<const uint4*>(g1 + off);
      g2v[k] = g2 ? *reinterpret_cast<const uint4*>(g2 + off) : make_uint4(0, 0, 0, 0);
      iv[k] = *reinterpret_cast<const uint2*>(idx + off);
    }
    V8 acc[4] = {};                       // [py * 2 + px]
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (!ok[k]) continue;
      const int dy = k >> 1, dxw = k & 1;
      const __nv_bfloat162* hg = reinterpret_cast<const __nv_bfloat162*>(&gv[k]);
      const __nv_bfloat162* hg2 = reinterpret_cast<const __nv_bfloat162*>(&g2v[k]);
      const uint8_t* ib = reinterpret_cast<const uint8_t*>(&iv[k]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = __bfloat1622float2(hg[j]);
        if (g2) {
          const float2 f2 = __bfloat1622float2(hg2[j]);
          f.x += f2.x;
          f.y += f2.y;
        }
#pragma unroll
        for (int py = 0; py < 2; ++py) {
          if (dy == 1 && py == 0) continue;
#pragma unroll
          for (int px = 0; px < 2; ++px) {
            if (dxw == 1 && px == 0) continue;
            const int pos = (py + 1 - 2 * dy) * 3 + (px + 1 - 2 * dxw);
            if (ib[2 * j] == pos) acc[py * 2 + px].v[2 * j] += f.x;
            if (ib[2 * j + 1] == pos) acc[py * 2 + px].v[2 * j + 1] += f.y;
          }
        }
      }
    }
#pragma unroll
    for (int py = 0; py < 2; ++py)
#pragma unroll
      for (int px = 0; px < 2; ++px)
        store8(dx + ((((int64_t)b * h + 2 * ya + py) * w + 2 * xb + px) * c + g * 8), acc[py * 2 + px]);
  }
}

// enc[b, c] = mean over hw pixels (fp32)            (nn.AvgPool2d(7) on a 7x7 map + view, resnet.py:137-138)
__global__ void avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, int n, int hw, int c, float* __restrict__ enc) {
  const int cg = c / 8;
  const int64_t total = (int64_t)n * cg;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const int b = (int)(i / cg);
    float acc[8] = {};
    for (int p = 0; p < hw; ++p) {
      const V8 v = load8(x + ((int64_t)b * hw + p) * c + g * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v.v[j];
    }
    const float inv = 1.f / (float)hw;
#pragma unroll
    for (int j = 0; j < 8; ++j) enc[(int64_t)b * c + g * 8 + j] = acc[j] * inv;
  }
}

__global__ void avgpool_bwd_kernel(const float* __restrict__ genc, int n, int hw, int c, __nv_bfloat16* __restrict__ dx) {
  const int cg = c / 8;
  const int64_t total = (int64_t)n * hw * cg;
  const float inv = 1.f / (float)hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const int b = (int)(i / ((int64_t)cg * hw));
    V8 o = loadf8(genc + (int64_t)b * c + g * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) o.v[j] *= inv;
    store8(dx + i * 8, o);
  }
}

// --------------------------------------------------------------- regressor
// pred[b] = dot(x[b,:], w) + bias          (nn.Linear(2048, 1), resnet.py:88,148)
__global__ void __launch_bounds__(256) linear1_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, int d,
                                                          float* __restrict__ pred) {
  __shared__ float sh[8];
  const int b = blockIdx.x;
  float acc = 0.f;
  for (int c = threadIdx.x; c < d; c += blockDim.x) acc = fmaf(x[(int64_t)b * d + c], w[c], acc);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += sh[i];
    pred[b] = t + bias[0];
  }
}

// dx[b,c] = g[b]*w[c];  dw[c] = sum_b g[b]*x[b,c];  dbias = sum_b g[b]     (thread per c)
__global__ void linear1_bwd_kernel(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ w,
                                   int n, int d, float* __restrict__ dx, float* __restrict__ dw,
                                   float* __restrict__ dbias) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  const float wc = w[c];
  float acc = 0.f, gb = 0.f;
  for (int b = 0; b < n; ++b) {
    const float gv = g[b];
    acc = fmaf(gv, x[(int64_t)b * d + c], acc);
    gb += gv;
    if (dx) dx[(int64_t)b * d + c] = gv * wc;
  }
  dw[c] = acc;
  if (c == 0) dbias[0] = gb;
}

// ---------------------------------------------------------------- optimizer
// torch.optim.Adam (no amsgrad; L2 weight decay added to the gradient), bias correction folded into step_size /
// bc2_sqrt on the host.  Flat fp32 buffers, 128-bit accesses.
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay, float bc1, float bc2_sqrt,
            float grad_scale, const float* __restrict__ clip_coef) {
  if (clip_coef) grad_scale *= clip_coef[0];
  const int64_t n4 = n / 4;
  const float step_size = lr / bc1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
    float* pa = &pp.x;
    const float* ga = &gg.x;
    float* ma = &mm.x;
    float* va = &vv.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float gr = ga[j] * grad_scale;
      if (weight_decay != 0.f) gr = fmaf(weight_decay, pa[j], gr);
      ma[j] = fmaf(beta1, ma[j], (1.f - beta1) * gr);
      va[j] = fmaf(beta2, va[j], (1.f - beta2) * gr * gr);
      const float denom = sqrtf(va[j]) / bc2_sqrt + eps;
      pa[j] -= step_size * (ma[j] / denom);
    }
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  // tail
  const int64_t i = n4 * 4 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) {
    float gr = g[i] * grad_scale;
    if (weight_decay != 0.f) gr = fmaf(weight_decay, p[i], gr);
    m[i] = fmaf(beta1, m[i], (1.f - beta1) * gr);
    v[i] = fmaf(beta2, v[i], (1.f - beta2) * gr * gr);
    p[i] -= step_size * (m[i] / (sqrtf(v[i]) / bc2_sqrt + eps));
  }
}

// One element of the multi-tensor Adam: adam_kernel's arithmetic with the last update written as one fma.  adam_kernel
// leaves `p -= step_size * q` to the compiler, which fuses it for some float4 lanes and not for others, so a parameter
// may differ from the flat step's by the rounding of step_size * q (about one ulp); m and v are the same bits.
__device__ __forceinline__ void adam_update(float& p, float gr, float& m, float& v, float beta1, float beta2, float eps,
                                            float weight_decay, float step_size, float bc2_sqrt) {
  if (weight_decay != 0.f) gr = fmaf(weight_decay, p, gr);
  m = fmaf(beta1, m, (1.f - beta1) * gr);
  v = fmaf(beta2, v, (1.f - beta2) * gr * gr);
  const float denom = sqrtf(v) / bc2_sqrt + eps;
  p = fmaf(-step_size, m / denom, p);
}

// Multi-tensor Adam: the segment table travels by value in the kernel's parameter block (no host-to-device copy, so a
// step is graph-capturable).  Each segment is cut into kAdamChunk-element chunks; chunk_start[s] is the first chunk of
// segment s and chunk_start[nseg] the total.  A CTA walks chunks grid-stride and finds each chunk's segment by binary
// search over the prefix.  Chunks start at multiples of 4 elements, so a segment whose four pointers are 16-byte aligned
// is read with float4s; any other segment (a view at a 4-byte offset) element by element.
constexpr int kAdamChunk = 4096;
constexpr int kAdamMultiMaxSegs = 512;

struct AdamMultiArgs {
  dirb200_adam_segment seg[kAdamMultiMaxSegs];
  int chunk_start[kAdamMultiMaxSegs + 1];
  int nseg;
  float lr, beta1, beta2, eps, weight_decay;
};
// CUDA >= 12.1 allows 32764 bytes of kernel parameters on sm_70 and newer
static_assert(sizeof(AdamMultiArgs) <= 32764, "adam_multi_kernel's parameter block is too large");

// kClip: every gradient is multiplied by the device scalar *clip_coef as it is read (clipping without rewriting
// .grad); without it the arithmetic is untouched, and a coefficient of exactly 1 gives the same bits.
template <bool kClip>
__global__ void __launch_bounds__(256) adam_multi_kernel(const __grid_constant__ AdamMultiArgs a,
                                                         const float* __restrict__ clip_coef) {
  const float coef = kClip ? *clip_coef : 1.f;
  const int total = a.chunk_start[a.nseg];
  for (int c = blockIdx.x; c < total; c += gridDim.x) {
    int lo = 0, hi = a.nseg - 1;                    // the last segment whose first chunk is <= c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (a.chunk_start[mid] <= c) lo = mid; else hi = mid - 1;
    }
    const dirb200_adam_segment& s = a.seg[lo];
    float* __restrict__ p = s.param;
    const float* __restrict__ g = s.grad;
    float* __restrict__ m = s.exp_avg;
    float* __restrict__ v = s.exp_avg_sq;
    const int64_t begin = (int64_t)(c - a.chunk_start[lo]) * kAdamChunk;
    const int64_t len = s.numel - begin < kAdamChunk ? s.numel - begin : kAdamChunk;
    const float step_size = a.lr / s.bc1, bc2_sqrt = s.bc2_sqrt;
    int64_t scalar_from = begin;
    if (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
          reinterpret_cast<uintptr_t>(v)) & 15) == 0) {
      const int n4 = (int)(len / 4);
      const int64_t b4 = begin / 4;
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 pp = reinterpret_cast<float4*>(p)[b4 + i];
        const float4 gg = reinterpret_cast<const float4*>(g)[b4 + i];
        float4 mm = reinterpret_cast<float4*>(m)[b4 + i], vv = reinterpret_cast<float4*>(v)[b4 + i];
        float* pa = &pp.x;
        const float* ga = &gg.x;
        float* ma = &mm.x;
        float* va = &vv.x;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          adam_update(pa[j], kClip ? ga[j] * coef : ga[j], ma[j], va[j], a.beta1, a.beta2, a.eps, a.weight_decay,
                      step_size, bc2_sqrt);
        reinterpret_cast<float4*>(p)[b4 + i] = pp;
        reinterpret_cast<float4*>(m)[b4 + i] = mm;
        reinterpret_cast<float4*>(v)[b4 + i] = vv;
      }
      scalar_from = begin + (int64_t)n4 * 4;
    }
    for (int64_t i = scalar_from + threadIdx.x; i < begin + len; i += blockDim.x) {
      float pi = p[i], mi = m[i], vi = v[i];
      adam_update(pi, kClip ? g[i] * coef : g[i], mi, vi, a.beta1, a.beta2, a.eps, a.weight_decay, step_size,
                  bc2_sqrt);
      m[i] = mi;
      v[i] = vi;
      p[i] = pi;
    }
  }
}

// torch.optim.SGD with momentum (dampening 0, no nesterov), weight decay
__global__ void __launch_bounds__(256)
sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, int64_t n, float lr,
           float momentum, float weight_decay, int first_step, float grad_scale, const float* __restrict__ clip_coef) {
  if (clip_coef) grad_scale *= clip_coef[0];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gr = g[i] * grad_scale;
    if (weight_decay != 0.f) gr = fmaf(weight_decay, p[i], gr);
    if (momentum != 0.f) {
      const float b = first_step ? gr : fmaf(momentum, buf[i], gr);
      buf[i] = b;
      gr = b;
    }
    p[i] -= lr * gr;
  }
}

// sum of (scale * g)^2 over the flat gradient: fp32 per thread, fp64 per block; the last block to finish (ticket)
// adds the block partials and writes the clip coefficient.
constexpr int kClipMaxGrid = 1024;
__global__ void __launch_bounds__(256)
grad_clip_kernel(const float* __restrict__ g, int64_t n, float scale, float max_norm, double* __restrict__ partials,
                 unsigned int* __restrict__ ticket, float* __restrict__ out) {
  __shared__ double sh[8];
  __shared__ bool last;
  float acc = 0.f;
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    acc = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, acc))));
  }
  if (blockIdx.x == 0)
    for (int64_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) acc = fmaf(g[i], g[i], acc);
  double t = warp_sum((double)acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += sh[w];
    partials[blockIdx.x] = s;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double tot = 0.0;
  for (int i = threadIdx.x; i < gridDim.x; i += blockDim.x) tot += ((volatile double*)partials)[i];
  tot = warp_sum(tot);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = tot;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += sh[w];
    const float norm = (float)(sqrt(s) * (double)fabsf(scale));
    const float coef = max_norm / (norm + 1e-6f);
    out[0] = coef < 1.f ? coef : 1.f;
    out[1] = norm;
    *ticket = 0u;                          // ready for the next step
  }
}

// Multi-tensor gradient norm: the (grad, numel) table travels by value, cut into kAdamChunk-element chunks as in
// adam_multi_kernel.  Each thread squares a chunk's elements in fp32 (at most kAdamChunk / 256 = 16 fmas) and adds
// that to an fp64 sum; CTA b adds its fp64 total into partials[b] (or writes it, in a call's first launch).  Every
// launch of one call uses the same grid, and launches on one stream run in order, so no atomics are needed for that.
// In the call's last launch the last CTA (ticket) sums partials[0 .. grid) in CTA order and writes {coef, norm}:
// two identical calls give identical bits.
struct GradNormArgs {
  const float* grad[kAdamMultiMaxSegs];
  int64_t numel[kAdamMultiMaxSegs];
  int chunk_start[kAdamMultiMaxSegs + 1];
  int nseg;
  int first, last;          // this launch is the call's first / last
  float max_norm;
};
static_assert(sizeof(GradNormArgs) <= 32764, "grad_norm_multi_kernel's parameter block is too large");

__global__ void __launch_bounds__(256) grad_norm_multi_kernel(const __grid_constant__ GradNormArgs a,
                                                              double* __restrict__ partials,
                                                              unsigned int* __restrict__ ticket,
                                                              float* __restrict__ out) {
  __shared__ double sh[8];
  __shared__ bool last;
  double acc = 0.0;
  const int total = a.chunk_start[a.nseg];
  for (int c = blockIdx.x; c < total; c += gridDim.x) {
    int lo = 0, hi = a.nseg - 1;                    // the last segment whose first chunk is <= c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (a.chunk_start[mid] <= c) lo = mid; else hi = mid - 1;
    }
    const float* __restrict__ g = a.grad[lo];
    const int64_t begin = (int64_t)(c - a.chunk_start[lo]) * kAdamChunk;
    const int64_t len = a.numel[lo] - begin < kAdamChunk ? a.numel[lo] - begin : kAdamChunk;
    float s = 0.f;
    int64_t scalar_from = begin;
    if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
      const int n4 = (int)(len / 4);
      const int64_t b4 = begin / 4;
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = reinterpret_cast<const float4*>(g)[b4 + i];
        s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s))));
      }
      scalar_from = begin + (int64_t)n4 * 4;
    }
    for (int64_t i = scalar_from + threadIdx.x; i < begin + len; i += blockDim.x) s = fmaf(g[i], g[i], s);
    acc += (double)s;
  }
  double t = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += sh[w];
    partials[blockIdx.x] = a.first ? s : partials[blockIdx.x] + s;
    if (a.last) {
      __threadfence();
      last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    } else {
      last = false;
    }
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double tot = 0.0;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) tot += ((volatile double*)partials)[i];
  tot = warp_sum(tot);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = tot;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += sh[w];
    const float norm = (float)sqrt(s);
    const float coef = a.max_norm / (norm + 1e-6f);
    out[0] = coef < 1.f ? coef : (coef == coef ? 1.f : coef);   // torch.clamp(coef, max=1) keeps a NaN
    out[1] = norm;
    *ticket = 0u;                          // ready for the next call
  }
}

static inline int grid1d(int64_t n, int block = 256, int per_sm = 8) {
  int64_t g = (n + block - 1) / block;
  const int64_t cap = (int64_t)per_sm * num_sms();
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// grid of the row-walking elementwise kernels: ~4 rows per thread, at most 8 CTAs per SM
static inline int stream_grid(int64_t rows, int lanes) {
  int64_t g = (rows + (int64_t)lanes * 4 - 1) / ((int64_t)lanes * 4);
  const int64_t cap = 8 * (int64_t)num_sms();
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// also holds the [CTA][2][c] rows of a conv epilogue: max(SMs, c / 64) CTAs
int bn_partial_floats(int max_c) {
  const int rows = kReduceCtasPerSm * num_sms() * 3, conv_rows = 2 * (max_c / 64);
  return (rows > conv_rows ? rows : conv_rows) * max_c;
}

static inline int reduce_grid(int64_t rows, int lanes, int ctas_per_sm = kReduceCtasPerSm) {
  int64_t g = (rows + (int64_t)lanes * 16 - 1) / ((int64_t)lanes * 16);   // >= ~16 rows per thread
  if (ctas_per_sm > kReduceCtasPerSm) ctas_per_sm = kReduceCtasPerSm;     // the partial buffer holds 4 rows per SM
  const int64_t cap = ctas_per_sm * (int64_t)num_sms();
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// CTAs of `kernel` (256 threads, `smem` dynamic bytes) that fit on one SM: the row-walking kernels are launched with
// exactly one resident wave (a grid of 4 x SMs on a kernel that fits 3 per SM runs a second, one-third-full wave).
template <typename K>
static int resident_ctas(K kernel, size_t smem) {
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, 256, smem) != cudaSuccess || occ < 1) {
    (void)cudaGetLastError();
    occ = 2;
  }
  return occ;
}

// ------------------------------------------------------------- host wrappers
// Channel counts of the row-walking BN kernels: a CTA's 256 threads are (c / 8 channel groups) x (row lanes), so c / 8
// must divide 256: c = 8, 16, 32, ..., 2048.  Tested before anything divides by c / 8.
static inline bool bn_channels_ok(int c) { return c >= 8 && c % 8 == 0 && 256 % (c / 8) == 0; }
// Compact second gradient (g2_h, g2_w > 0): even maps that tile the rows; CompactG2::locate divides 32-bit row indices.
static inline bool compact_ok(int g2_h, int g2_w, int64_t rows) {
  if (g2_h == 0 && g2_w == 0) return true;
  return g2_h > 0 && g2_w > 0 && g2_h % 2 == 0 && g2_w % 2 == 0 && rows < (int64_t(1) << 31) &&
         rows % ((int64_t)g2_h * g2_w) == 0;
}

int bn_stats(const __nv_bfloat16* y, int64_t rows, int c, float* partial, int* nblocks, cudaStream_t st) {
  DIRB_CHECK_ARG(bn_channels_ok(c), "bn_stats: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0, "bn_stats: rows must be positive");
  const int cgroups = c / 8;
  const int lanes = 256 / cgroups;
  *nblocks = reduce_grid(rows, lanes);
  bn_stats_kernel<<<*nblocks, 256, 256 * 16 * sizeof(float), st>>>(y, rows, c, partial);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_finalize(const float* partial, const StatLayout& layout, int64_t rows, int c, const float* gamma,
                const float* beta, float eps, float momentum, float* running_mean, float* running_var, float* mean,
                float* invstd, float* scale, float* shift, cudaStream_t st) {
  DIRB_CHECK_ARG(layout.rows > 0 && layout.n_tiles > 0 && layout.bn > 0 && layout.group > 0 &&
                     layout.n_tiles * layout.bn >= c,
                 "bn_finalize: bad statistics layout");
  bn_finalize_kernel<<<(c + 31) / 32, dim3(32, 32), 0, st>>>(partial, layout, rows, c, gamma, beta, eps, momentum,
                                                             running_mean, running_var, mean, invstd, scale, shift);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_eval_coeffs(int c, const float* gamma, const float* beta, float eps, const float* running_mean,
                   const float* running_var, float* scale, float* shift, cudaStream_t st) {
  bn_eval_coeffs_kernel<<<(c + 127) / 128, 128, 0, st>>>(c, gamma, beta, eps, running_mean, running_var, scale, shift);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_eval_coeffs_all(const BnEvalDesc* descs_dev, int nlayers, int max_c, const float* params, const float* running,
                       float eps, cudaStream_t st) {
  bn_eval_coeffs_all_kernel<<<dim3((max_c + 255) / 256, nlayers), 256, 0, st>>>(descs_dev, params, running, eps);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_apply(const __nv_bfloat16* y, const float* scale, const float* shift, const __nv_bfloat16* res,
             const __nv_bfloat16* res_y, const float* res_scale, const float* res_shift, bool relu, int64_t rows, int c,
             __nv_bfloat16* out, uint8_t* mask_out, cudaStream_t st) {
  DIRB_CHECK_ARG(bn_channels_ok(c), "bn_apply: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0, "bn_apply: rows must be positive");
  const int cgroups = c / 8;
  DIRB_CHECK_ARG(!(res && res_y), "bn_apply: one shortcut operand (identity or the downsample branch's raw output)");
  // the mask bit tests the stored value for a non-zero magnitude: that is "> 0" only behind the ReLU
  DIRB_CHECK_ARG(!mask_out || relu, "bn_apply: the ReLU mask needs relu");
  const int want = stream_grid(rows, 256 / cgroups);
#define DIRB_BNA(RES, RESY, MASK)                                                                                 \
  do {                                                                                                            \
    static const int occ = resident_ctas(bn_apply_kernel<RES, RESY, MASK>, 0);                                    \
    const int grid = want < occ * num_sms() ? want : occ * num_sms();                                             \
    bn_apply_kernel<RES, RESY, MASK><<<grid, 256, 0, st>>>(y, scale, shift, res, res_y, res_scale, res_shift,     \
                                                           relu ? 1 : 0, rows, c, out, mask_out);                 \
  } while (0)
  if (res && mask_out) DIRB_BNA(true, false, true);
  else if (res) DIRB_BNA(true, false, false);
  else if (res_y && mask_out) DIRB_BNA(false, true, true);
  else if (res_y) DIRB_BNA(false, true, false);
  else if (mask_out) DIRB_BNA(false, false, true);
  else DIRB_BNA(false, false, false);
#undef DIRB_BNA
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

// mask == nullptr: conv -> BN -> ReLU layer, the ReLU mask is re-derived from y with (scale, shift);
// mask != nullptr: block output, the bit mask bn_apply stored (g2 / y2: second incoming gradient / downsample branch).
static CompactG2 make_compact(int g2_h, int g2_w) {
  CompactG2 cg{};
  if (g2_h > 0 && g2_w > 0) {
    cg.hw = make_fastdiv(static_cast<uint32_t>(g2_h) * g2_w);
    cg.w = make_fastdiv(static_cast<uint32_t>(g2_w));
    cg.h2 = g2_h / 2;
    cg.w2 = g2_w / 2;
  }
  return cg;
}

// g2_h, g2_w > 0: g2 is the compact [n, g2_h/2, g2_w/2, c] tensor (rows are the pixels of the g2_h x g2_w maps)
int bn_bwd_reduce(const __nv_bfloat16* g1, const __nv_bfloat16* g2, const __nv_bfloat16* y, const __nv_bfloat16* y2,
                  const float* scale, const float* shift, const uint8_t* mask, int64_t rows, int c, float* partial,
                  int* nblocks, cudaStream_t st, int g2_h, int g2_w, __nv_bfloat16* dz_out, const __nv_bfloat16* g3) {
  const CompactG2 cg2 = make_compact(g2_h, g2_w);
  DIRB_CHECK_ARG(!g3 || (g2 && dz_out), "bn_bwd_reduce: a third gradient is added in the two-gradient identity forms only");
  DIRB_CHECK_ARG(bn_channels_ok(c), "bn_bwd_reduce: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0, "bn_bwd_reduce: rows must be positive");
  DIRB_CHECK_ARG(compact_ok(g2_h, g2_w, rows) && (g2_h == 0 || (g2 && mask && !y2)),
                 "bn_bwd_reduce: bad compact second gradient");
  const int cgroups = c / 8;
  DIRB_CHECK_ARG(mask || (!g2 && !y2 && (scale != nullptr) == (shift != nullptr)),
                 "bn_bwd_reduce: the mask-from-y and the no-ReLU forms take one gradient, one BN");
  DIRB_CHECK_ARG(!dz_out || (mask && !y2), "bn_bwd_reduce: dz is stored for identity blocks only");
  const int lanes = 256 / cgroups;
  const size_t smem = 256 * (y2 ? 24 : 16) * sizeof(float);
#define DIRB_RED3(MODE, G2, Y2, DZ, G3)                                                                             \
  do {                                                                                                              \
    static const int occ = resident_ctas(bn_bwd_reduce_kernel<MODE, G2, Y2, DZ, G3>, 256 * 24 * sizeof(float));     \
    *nblocks = reduce_grid(rows, lanes, occ);                                                                       \
    bn_bwd_reduce_kernel<MODE, G2, Y2, DZ, G3><<<*nblocks, 256, smem, st>>>(g1, g2, cg2, g3, y, y2, scale, shift, mask, \
                                                                            rows, c, partial, dz_out);              \
  } while (0)
#define DIRB_RED(MODE, G2, Y2, DZ) DIRB_RED3(MODE, G2, Y2, DZ, false)
  if (g3 && g2_h) DIRB_RED3(MASK_BITS, G2_COMPACT, false, true, true);
  else if (g3) DIRB_RED3(MASK_BITS, G2_DENSE, false, true, true);
  else if (!mask && !scale) DIRB_RED(MASK_NONE, G2_NONE, false, false);   // BN without a ReLU behind it
  else if (!mask) DIRB_RED(MASK_FROM_Y, G2_NONE, false, false);
  else if (g2_h && dz_out) DIRB_RED(MASK_BITS, G2_COMPACT, false, true);
  else if (g2_h) DIRB_RED(MASK_BITS, G2_COMPACT, false, false);
  else if (g2 && y2) DIRB_RED(MASK_BITS, G2_DENSE, true, false);
  else if (g2 && dz_out) DIRB_RED(MASK_BITS, G2_DENSE, false, true);
  else if (g2) DIRB_RED(MASK_BITS, G2_DENSE, false, false);
  else if (y2) DIRB_RED(MASK_BITS, G2_NONE, true, false);
  else if (dz_out) DIRB_RED(MASK_BITS, G2_NONE, false, true);
  else DIRB_RED(MASK_BITS, G2_NONE, false, false);
#undef DIRB_RED
#undef DIRB_RED3
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_bwd_coeffs(const float* partial, int nblocks, int k, int gslot, int64_t rows, int c, const float* mean,
                  const float* invstd, const float* gamma, float* grad_gamma, float* grad_beta, float* coef,
                  cudaStream_t st) {
  bn_bwd_coeffs_kernel<<<(c + 31) / 32, dim3(32, 32), 0, st>>>(partial, nblocks, k, gslot, rows, c, mean, invstd, gamma,
                                                      grad_gamma, grad_beta, coef);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_bwd_coeffs_layout(const float* partial, const StatLayout& layout, int64_t rows, int c, const float* mean,
                         const float* invstd, const float* gamma, float* grad_gamma, float* grad_beta, float* coef,
                         cudaStream_t st) {
  DIRB_CHECK_ARG(layout.rows > 0 && layout.n_tiles > 0 && layout.bn > 0 && layout.group > 0 &&
                     layout.n_tiles * layout.bn >= c,
                 "bn_bwd_coeffs_layout: bad partial layout");
  bn_bwd_coeffs_layout_kernel<<<(c + 31) / 32, dim3(32, 32), 0, st>>>(partial, layout, rows, c, mean, invstd, gamma,
                                                                      grad_gamma, grad_beta, coef);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_bwd_apply(const __nv_bfloat16* g1, const __nv_bfloat16* g2, const __nv_bfloat16* y, const float* coef,
                 const __nv_bfloat16* y2, const float* coef2, const float* scale, const float* shift,
                 const uint8_t* mask, int64_t rows, int c, __nv_bfloat16* dy, __nv_bfloat16* dy2,
                 __nv_bfloat16* dz_out, cudaStream_t st, int g2_h, int g2_w) {
  const CompactG2 cg2 = make_compact(g2_h, g2_w);
  DIRB_CHECK_ARG(bn_channels_ok(c), "bn_bwd_apply: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0, "bn_bwd_apply: rows must be positive");
  DIRB_CHECK_ARG(compact_ok(g2_h, g2_w, rows) && (g2_h == 0 || (g2 && mask && !y2 && dz_out)),
                 "bn_bwd_apply: bad compact second gradient");
  const int cgroups = c / 8;
  DIRB_CHECK_ARG(mask || (!g2 && !y2 && !dz_out && (scale != nullptr) == (shift != nullptr)),
                 "bn_bwd_apply: the mask-from-y and the dz-input forms take one gradient, one BN");
  DIRB_CHECK_ARG(!(y2 && dz_out), "bn_bwd_apply: a block has either a downsample branch or an identity path");
  const int want = stream_grid(rows, 256 / cgroups);
#define DIRB_APP(MODE, G2, Y2, DZ)                                                                                     \
  do {                                                                                                                 \
    static const int occ = resident_ctas(bn_bwd_apply_kernel<MODE, G2, Y2, DZ>, 0);                                    \
    const int grid = want < occ * num_sms() ? want : occ * num_sms();                                                  \
    bn_bwd_apply_kernel<MODE, G2, Y2, DZ><<<grid, 256, 0, st>>>(g1, g2, cg2, y, coef, y2, coef2, scale, shift, mask, rows, \
                                                               c, dy, dy2, dz_out);                                    \
  } while (0)
  if (!mask && !scale) DIRB_APP(MASK_NONE, G2_NONE, false, false);     // g1 is dz already (bn_bwd_reduce stored it)
  else if (!mask) DIRB_APP(MASK_FROM_Y, G2_NONE, false, false);
  else if (g2_h) DIRB_APP(MASK_BITS, G2_COMPACT, false, true);
  else if (g2 && y2) DIRB_APP(MASK_BITS, G2_DENSE, true, false);
  else if (g2 && dz_out) DIRB_APP(MASK_BITS, G2_DENSE, false, true);
  else if (g2) DIRB_APP(MASK_BITS, G2_DENSE, false, false);
  else if (y2) DIRB_APP(MASK_BITS, G2_NONE, true, false);
  else if (dz_out) DIRB_APP(MASK_BITS, G2_NONE, false, true);
  else DIRB_APP(MASK_BITS, G2_NONE, false, false);
#undef DIRB_APP
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int maxpool_fwd(const __nv_bfloat16* x, int n, int h, int w, int c, __nv_bfloat16* out, uint8_t* idx, cudaStream_t st) {
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  maxpool_fwd_kernel<<<grid1d((int64_t)n * ho * wo * c / 8), 256, 0, st>>>(x, n, h, w, c, out, idx);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bn_relu_maxpool_fwd(const __nv_bfloat16* y, const float* scale, const float* shift, int n, int h, int w, int c,
                        __nv_bfloat16* out, uint8_t* idx, cudaStream_t st) {
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  bn_relu_maxpool_fwd_kernel<<<grid1d((int64_t)n * ((ho + 1) / 2) * ((wo + 1) / 2) * c / 8), 256, 0, st>>>(y, scale, shift, n, h, w, c,
                                                                                                out, idx);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int maxpool_bwd(const __nv_bfloat16* g1, const __nv_bfloat16* g2, const uint8_t* idx, int n, int h, int w, int c,
                __nv_bfloat16* dx, cudaStream_t st) {
  DIRB_CHECK_ARG(h % 2 == 0 && w % 2 == 0, "maxpool_bwd: H and W must be even");
  maxpool_bwd_kernel<<<grid1d((int64_t)n * (h / 2) * (w / 2) * c / 8), 256, 0, st>>>(g1, g2, idx, n, h, w, c, dx);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int avgpool_fwd(const __nv_bfloat16* x, int n, int hw, int c, float* enc, cudaStream_t st) {
  avgpool_fwd_kernel<<<grid1d((int64_t)n * c / 8, 128), 128, 0, st>>>(x, n, hw, c, enc);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int avgpool_bwd(const float* genc, int n, int hw, int c, __nv_bfloat16* dx, cudaStream_t st) {
  avgpool_bwd_kernel<<<grid1d((int64_t)n * hw * c / 8), 256, 0, st>>>(genc, n, hw, c, dx);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // namespace dirb200

using namespace dirb200;

extern "C" {

/* ---- BatchNorm2d (training mode) / pooling on NHWC bf16 tensors: the layers between the convolutions, as entry points
 * of their own (the ResNet runner sequences the same kernels internally; the NYUD2 decoder modules need them singly). */
size_t dirb200_bn_workspace_bytes(int c) { return sizeof(float) * static_cast<size_t>(bn_partial_floats(c)); }

int dirb200_bn_train_fwd(const void* y, int64_t rows, int c, const float* gamma, const float* beta, float eps,
                         float momentum, float* running_mean, float* running_var, int relu, void* out, float* save_mean,
                         float* save_invstd, float* scale_shift, void* workspace, void* stream) {
  DIRB_CHECK_ARG(y && out && gamma && beta && save_mean && save_invstd && scale_shift && workspace,
                 "bn_train_fwd: null pointer");
  DIRB_CHECK_ARG(bn_channels_ok(c), "bn_train_fwd: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0, "bn_train_fwd: rows must be positive");
  cudaStream_t st = as_stream(stream);
  float* partial = static_cast<float*>(workspace);
  int nblk = 0;
  if (int rc = bn_stats(static_cast<const __nv_bfloat16*>(y), rows, c, partial, &nblk, st)) return rc;
  if (int rc = bn_finalize(partial, StatLayout{nblk, 1, c, 1}, rows, c, gamma, beta, eps, momentum, running_mean, running_var,
                           save_mean, save_invstd, scale_shift, scale_shift + c, st))
    return rc;
  return bn_apply(static_cast<const __nv_bfloat16*>(y), scale_shift, scale_shift + c, nullptr, nullptr, nullptr, nullptr,
                  relu != 0, rows, c, static_cast<__nv_bfloat16*>(out), nullptr, st);
}

int dirb200_bn_train_bwd(const void* grad_out, const void* y, int64_t rows, int c, const float* gamma,
                         const float* save_mean, const float* save_invstd, const float* scale_shift, int relu,
                         float* grad_gamma, float* grad_beta, void* grad_y, void* workspace, void* stream) {
  DIRB_CHECK_ARG(grad_out && y && gamma && save_mean && save_invstd && grad_gamma && grad_beta && grad_y && workspace &&
                     (!relu || scale_shift),
                 "bn_train_bwd: null pointer");
  // before bn_partial_floats(c) below: it queries the device
  DIRB_CHECK_ARG(bn_channels_ok(c), "bn_train_bwd: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0, "bn_train_bwd: rows must be positive");
  cudaStream_t st = as_stream(stream);
  float* partial = static_cast<float*>(workspace);
  float* coef = partial + bn_partial_floats(c) - 3 * c;        // the reduction uses at most 2/3 of the buffer
  const float* sc = relu ? scale_shift : nullptr;
  const float* sh = relu ? scale_shift + c : nullptr;
  int nblk = 0;
  if (int rc = bn_bwd_reduce(static_cast<const __nv_bfloat16*>(grad_out), nullptr, static_cast<const __nv_bfloat16*>(y),
                             nullptr, sc, sh, nullptr, rows, c, partial, &nblk, st))
    return rc;
  if (int rc = bn_bwd_coeffs(partial, nblk, 2, 1, rows, c, save_mean, save_invstd, gamma, grad_gamma, grad_beta, coef, st))
    return rc;
  return bn_bwd_apply(static_cast<const __nv_bfloat16*>(grad_out), nullptr, static_cast<const __nv_bfloat16*>(y), coef,
                      nullptr, nullptr, sc, sh, nullptr, rows, c, static_cast<__nv_bfloat16*>(grad_y), nullptr, nullptr, st);
}

int dirb200_bn_eval_coeffs(int c, const float* gamma, const float* beta, float eps, const float* running_mean,
                           const float* running_var, float* scale, float* shift, void* stream) {
  DIRB_CHECK_ARG(gamma && beta && running_mean && running_var && scale && shift, "bn_eval_coeffs: null pointer");
  DIRB_CHECK_ARG(c > 0, "bn_eval_coeffs: c must be positive");
  return bn_eval_coeffs(c, gamma, beta, eps, running_mean, running_var, scale, shift, as_stream(stream));
}

/* Test aid: the runner's one-launch eval coefficients of every BatchNorm, over caller-given jobs (see include/dirb200.h). */
int dirb200_bn_eval_coeffs_all(const dirb200_bn_eval_job* jobs_host, int njobs, const float* params,
                               const float* running, float eps, void* stream) {
  DIRB_CHECK_ARG(jobs_host && params && running, "bn_eval_coeffs_all: null pointer");
  DIRB_CHECK_ARG(njobs >= 1 && njobs <= 65535, "bn_eval_coeffs_all: njobs must be 1 .. 65535 (got %d)", njobs);
  std::vector<BnEvalDesc> descs;
  int max_c = 0;
  for (int k = 0; k < njobs; ++k) {
    const dirb200_bn_eval_job& j = jobs_host[k];
    DIRB_CHECK_ARG(j.scale && j.shift, "bn_eval_coeffs_all: job %d has a null scale or shift", k);
    DIRB_CHECK_ARG(j.c > 0, "bn_eval_coeffs_all: job %d has a non-positive channel count %d", k, j.c);
    DIRB_CHECK_ARG(j.gamma_off >= 0 && j.beta_off >= 0 && j.rm_off >= 0 && j.rv_off >= 0,
                   "bn_eval_coeffs_all: job %d has a negative offset", k);
    descs.push_back(BnEvalDesc{j.c, (size_t)j.gamma_off, (size_t)j.beta_off, (size_t)j.rm_off, (size_t)j.rv_off, j.scale,
                               j.shift});
    if (j.c > max_c) max_c = j.c;
  }
  cudaStream_t st = as_stream(stream);
  return with_device_table(descs, st, [&](const BnEvalDesc* d) {
    return bn_eval_coeffs_all(d, njobs, max_c, params, running, eps, st);
  });
}

/* ---- Test aids: the consumers of the per-CTA rows the conv epilogues write (see include/dirb200.h). */
int dirb200_bn_finalize_layout(const float* partial, const int* layout_host, int64_t rows, int c, const float* gamma,
                               const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                               float* mean_out, float* invstd_out, float* scale_out, float* shift_out, void* stream) {
  DIRB_CHECK_ARG(partial && layout_host && gamma && beta && mean_out && invstd_out && scale_out && shift_out && rows > 0 &&
                     c > 0 && (running_mean == nullptr) == (running_var == nullptr),
                 "bn_finalize_layout: null pointer or bad size");
  const StatLayout lay{layout_host[0], layout_host[1], layout_host[2], layout_host[3]};
  return bn_finalize(partial, lay, rows, c, gamma, beta, eps, momentum, running_mean, running_var, mean_out, invstd_out,
                     scale_out, shift_out, as_stream(stream));
}

int dirb200_bn_bwd_coeffs_layout(const float* partial, const int* layout_host, int64_t rows, int c, const float* mean,
                                 const float* invstd, const float* gamma, float* grad_gamma, float* grad_beta,
                                 float* coef_out, void* stream) {
  DIRB_CHECK_ARG(partial && layout_host && mean && invstd && gamma && grad_gamma && grad_beta && coef_out && rows > 0 &&
                     c > 0,
                 "bn_bwd_coeffs_layout: null pointer or bad size");
  const StatLayout lay{layout_host[0], layout_host[1], layout_host[2], layout_host[3]};
  return bn_bwd_coeffs_layout(partial, lay, rows, c, mean, invstd, gamma, grad_gamma, grad_beta, coef_out,
                              as_stream(stream));
}

/* ---- Test aids: the BatchNorm / pooling layer kernels, one launch each (see include/dirb200.h).  The internal
 * wrappers refuse unsupported channel counts, row counts and operand combinations before their first CUDA call; these
 * add the pointer checks. */
using bf16 = __nv_bfloat16;

int dirb200_layer_bn_stats(const void* y, int64_t rows, int c, float* partial, int* nblocks_host, void* stream) {
  DIRB_CHECK_ARG(y && partial && nblocks_host, "layer_bn_stats: null pointer");
  return bn_stats(static_cast<const bf16*>(y), rows, c, partial, nblocks_host, as_stream(stream));
}

int dirb200_layer_bn_apply(const void* y, const float* scale, const float* shift, const void* res, const void* res_y,
                           const float* res_scale, const float* res_shift, int relu, int64_t rows, int c, void* out,
                           uint8_t* mask_out, void* stream) {
  DIRB_CHECK_ARG(y && scale && shift && out, "layer_bn_apply: null pointer");
  DIRB_CHECK_ARG(!res_y || (res_scale && res_shift), "layer_bn_apply: res_y needs res_scale and res_shift");
  return bn_apply(static_cast<const bf16*>(y), scale, shift, static_cast<const bf16*>(res), static_cast<const bf16*>(res_y),
                  res_scale, res_shift, relu != 0, rows, c, static_cast<bf16*>(out), mask_out, as_stream(stream));
}

int dirb200_layer_bn_bwd_reduce(const void* g1, const void* g2, const void* g3, const void* y, const void* y2,
                                const float* scale, const float* shift, const uint8_t* mask, int64_t rows, int c,
                                int g2_h, int g2_w, void* dz_out, float* partial, int* nblocks_host, void* stream) {
  DIRB_CHECK_ARG(g1 && y && partial && nblocks_host, "layer_bn_bwd_reduce: null pointer");
  return bn_bwd_reduce(static_cast<const bf16*>(g1), static_cast<const bf16*>(g2), static_cast<const bf16*>(y),
                       static_cast<const bf16*>(y2), scale, shift, mask, rows, c, partial, nblocks_host,
                       as_stream(stream), g2_h, g2_w, static_cast<bf16*>(dz_out), static_cast<const bf16*>(g3));
}

int dirb200_layer_bn_bwd_coeffs(const float* partial, int nblocks, int k, int gslot, int64_t rows, int c,
                                const float* mean, const float* invstd, const float* gamma, float* grad_gamma,
                                float* grad_beta, float* coef_out, void* stream) {
  DIRB_CHECK_ARG(partial && mean && invstd && gamma && grad_gamma && grad_beta && coef_out,
                 "layer_bn_bwd_coeffs: null pointer");
  DIRB_CHECK_ARG(bn_channels_ok(c), "layer_bn_bwd_coeffs: unsupported channel count %d (8, 16, 32, ..., 2048)", c);
  DIRB_CHECK_ARG(rows > 0 && nblocks > 0, "layer_bn_bwd_coeffs: rows and nblocks must be positive");
  DIRB_CHECK_ARG((k == 2 || k == 3) && gslot >= 1 && gslot < k, "layer_bn_bwd_coeffs: K must be 2 or 3, 1 <= gslot < K");
  return bn_bwd_coeffs(partial, nblocks, k, gslot, rows, c, mean, invstd, gamma, grad_gamma, grad_beta, coef_out,
                       as_stream(stream));
}

int dirb200_layer_bn_bwd_apply(const void* g1, const void* g2, const void* y, const float* coef, const void* y2,
                               const float* coef2, const float* scale, const float* shift, const uint8_t* mask,
                               int64_t rows, int c, int g2_h, int g2_w, void* dy, void* dy2, void* dz_out,
                               void* stream) {
  DIRB_CHECK_ARG(g1 && y && coef && dy, "layer_bn_bwd_apply: null pointer");
  DIRB_CHECK_ARG(!y2 || (coef2 && dy2), "layer_bn_bwd_apply: y2 needs coef2 and dy2");
  return bn_bwd_apply(static_cast<const bf16*>(g1), static_cast<const bf16*>(g2), static_cast<const bf16*>(y), coef,
                      static_cast<const bf16*>(y2), coef2, scale, shift, mask, rows, c, static_cast<bf16*>(dy),
                      static_cast<bf16*>(dy2), static_cast<bf16*>(dz_out), as_stream(stream), g2_h, g2_w);
}

int dirb200_layer_bn_relu_maxpool_fwd(const void* y, const float* scale, const float* shift, int n, int h, int w, int c,
                                      void* out, uint8_t* argmax, void* stream) {
  DIRB_CHECK_ARG(y && scale && shift && out && argmax, "layer_bn_relu_maxpool_fwd: null pointer");
  DIRB_CHECK_ARG(n > 0 && h > 0 && w > 0, "layer_bn_relu_maxpool_fwd: bad map size");
  DIRB_CHECK_ARG(c > 0 && c % 8 == 0, "layer_bn_relu_maxpool_fwd: unsupported channel count %d (a multiple of 8)", c);
  return bn_relu_maxpool_fwd(static_cast<const bf16*>(y), scale, shift, n, h, w, c, static_cast<bf16*>(out), argmax,
                             as_stream(stream));
}

int dirb200_layer_maxpool_bwd(const void* g1, const void* g2, const uint8_t* argmax, int n, int h, int w, int c,
                              void* dx, void* stream) {
  DIRB_CHECK_ARG(g1 && argmax && dx, "layer_maxpool_bwd: null pointer");
  DIRB_CHECK_ARG(n > 0 && h > 0 && w > 0, "layer_maxpool_bwd: bad map size");
  DIRB_CHECK_ARG(c > 0 && c % 8 == 0, "layer_maxpool_bwd: unsupported channel count %d (a multiple of 8)", c);
  return maxpool_bwd(static_cast<const bf16*>(g1), static_cast<const bf16*>(g2), argmax, n, h, w, c,
                     static_cast<bf16*>(dx), as_stream(stream));
}

int dirb200_maxpool3x3s2_fwd(const void* x, int n, int h, int w, int c, void* out, uint8_t* argmax, void* stream) {
  DIRB_CHECK_ARG(x && out && argmax && n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "maxpool_fwd: bad arguments");
  return maxpool_fwd(static_cast<const __nv_bfloat16*>(x), n, h, w, c, static_cast<__nv_bfloat16*>(out), argmax,
                     as_stream(stream));
}

int dirb200_maxpool3x3s2_bwd(const void* grad_out, const uint8_t* argmax, int n, int h, int w, int c, void* grad_x,
                             void* stream) {
  DIRB_CHECK_ARG(grad_out && argmax && grad_x && n > 0 && c > 0 && c % 8 == 0, "maxpool_bwd: bad arguments");
  return maxpool_bwd(static_cast<const __nv_bfloat16*>(grad_out), nullptr, argmax, n, h, w, c,
                     static_cast<__nv_bfloat16*>(grad_x), as_stream(stream));
}

int dirb200_avgpool_fwd(const void* x, int n, int hw, int c, float* out, void* stream) {
  DIRB_CHECK_ARG(x && out && n > 0 && hw > 0 && c > 0 && c % 8 == 0, "avgpool_fwd: bad arguments");
  return avgpool_fwd(static_cast<const __nv_bfloat16*>(x), n, hw, c, out, as_stream(stream));
}

int dirb200_avgpool_bwd(const float* grad_out, int n, int hw, int c, void* grad_x, void* stream) {
  DIRB_CHECK_ARG(grad_out && grad_x && n > 0 && hw > 0 && c > 0 && c % 8 == 0, "avgpool_bwd: bad arguments");
  return avgpool_bwd(grad_out, n, hw, c, static_cast<__nv_bfloat16*>(grad_x), as_stream(stream));
}

int dirb200_linear1_fwd(const float* x, const float* w, const float* bias, int64_t n, int d, float* pred,
                        void* stream) {
  // one CTA per row: n is the grid size
  DIRB_CHECK_ARG(x && w && bias && pred && n > 0 && n <= INT32_MAX && d > 0, "linear1_fwd: bad arguments");
  linear1_fwd_kernel<<<(unsigned)n, 256, 0, as_stream(stream)>>>(x, w, bias, d, pred);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_linear1_bwd(const float* grad_pred, const float* x, const float* w, int64_t n, int d, float* dx,
                        float* dw, float* dbias, void* stream) {
  // the kernel walks the n rows with a 32-bit counter
  DIRB_CHECK_ARG(grad_pred && x && w && dw && dbias && n > 0 && n <= INT32_MAX && d > 0, "linear1_bwd: bad arguments");
  linear1_bwd_kernel<<<(d + 127) / 128, 128, 0, as_stream(stream)>>>(grad_pred, x, w, (int)n, d, dx, dw, dbias);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                      float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                      const float* clip_coef, void* stream) {
  DIRB_CHECK_ARG(params && grads && exp_avg && exp_avg_sq && n > 0 && step >= 1, "adam_step: bad arguments");
  DIRB_CHECK_ARG((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) |
                  reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq)) % 16 == 0,
                 "adam_step: buffers must be 16-byte aligned");
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  adam_kernel<<<grid1d(n / 4 + 1), 256, 0, as_stream(stream)>>>(params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2,
                                                               eps, weight_decay, (float)bc1, (float)sqrt(bc2),
                                                               grad_scale, clip_coef);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

// dirb200_adam_step_multi and its clipped form: the checks, then one launch per kAdamMultiMaxSegs segments
static int adam_multi(const char* name, const dirb200_adam_segment* segs_host, int nseg, float lr, float beta1,
                      float beta2, float eps, float weight_decay, const float* clip_coef, void* stream) {
  DIRB_CHECK_ARG(segs_host && nseg > 0, "%s: bad arguments (segs_host %p, nseg %d)", name, (const void*)segs_host,
                 nseg);
  for (int k = 0; k < nseg; ++k) {
    const dirb200_adam_segment& s = segs_host[k];
    DIRB_CHECK_ARG(s.param && s.grad && s.exp_avg && s.exp_avg_sq, "%s: segment %d has a null pointer", name, k);
    DIRB_CHECK_ARG(((reinterpret_cast<uintptr_t>(s.param) | reinterpret_cast<uintptr_t>(s.grad) |
                     reinterpret_cast<uintptr_t>(s.exp_avg) | reinterpret_cast<uintptr_t>(s.exp_avg_sq)) & 3) == 0,
                   "%s: segment %d is not 4-byte aligned", name, k);
    DIRB_CHECK_ARG(s.numel > 0 && (s.numel - 1) / kAdamChunk < INT32_MAX,
                   "%s: segment %d has numel %lld (1 .. 2^31 chunks of %d)", name, k, (long long)s.numel,
                   kAdamChunk);
    DIRB_CHECK_ARG(isfinite(s.bc1) && s.bc1 > 0.f && isfinite(s.bc2_sqrt) && s.bc2_sqrt > 0.f,
                   "%s: segment %d has bias corrections bc1 %g, bc2_sqrt %g (finite and positive)", name, k,
                   (double)s.bc1, (double)s.bc2_sqrt);
  }
  AdamMultiArgs a;
  a.lr = lr;
  a.beta1 = beta1;
  a.beta2 = beta2;
  a.eps = eps;
  a.weight_decay = weight_decay;
  // a launch takes up to kAdamMultiMaxSegs segments, as long as its chunk count fits the int prefix
  for (int k = 0; k < nseg;) {
    int ns = 0;
    int64_t chunks = 0;
    a.chunk_start[0] = 0;
    while (k < nseg && ns < kAdamMultiMaxSegs) {
      const int64_t c = (segs_host[k].numel + kAdamChunk - 1) / kAdamChunk;
      if (ns > 0 && chunks + c > INT32_MAX) break;
      a.seg[ns] = segs_host[k];
      chunks += c;
      a.chunk_start[++ns] = (int)chunks;
      ++k;
    }
    a.nseg = ns;
    if (clip_coef)
      adam_multi_kernel<true><<<grid1d(chunks, 1), 256, 0, as_stream(stream)>>>(a, clip_coef);
    else
      adam_multi_kernel<false><<<grid1d(chunks, 1), 256, 0, as_stream(stream)>>>(a, nullptr);
    DIRB_LAUNCHED();
  }
  return DIRB200_OK;
}

int dirb200_adam_step_multi(const dirb200_adam_segment* segs_host, int nseg, float lr, float beta1, float beta2,
                            float eps, float weight_decay, void* stream) {
  return adam_multi("adam_step_multi", segs_host, nseg, lr, beta1, beta2, eps, weight_decay, nullptr, stream);
}

int dirb200_adam_step_multi_clipped(const dirb200_adam_segment* segs_host, int nseg, float lr, float beta1,
                                    float beta2, float eps, float weight_decay, const float* clip_coef,
                                    void* stream) {
  DIRB_CHECK_ARG(clip_coef, "adam_step_multi_clipped: clip_coef is null");
  return adam_multi("adam_step_multi_clipped", segs_host, nseg, lr, beta1, beta2, eps, weight_decay, clip_coef,
                    stream);
}

int dirb200_sgd_step(float* params, const float* grads, float* momentum_buf, int64_t n, float lr, float momentum,
                     float weight_decay, int first_step, float grad_scale, const float* clip_coef, void* stream) {
  DIRB_CHECK_ARG(params && grads && n > 0 && (momentum == 0.f || momentum_buf), "sgd_step: bad arguments");
  sgd_kernel<<<grid1d(n), 256, 0, as_stream(stream)>>>(params, grads, momentum_buf, n, lr, momentum, weight_decay,
                                                      first_step, grad_scale, clip_coef);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

size_t dirb200_grad_clip_workspace_bytes(void) { return sizeof(double) * kClipMaxGrid + 16; }

/* The workspace must be zero-initialised once (its ticket word is reset by the kernel after every use). */
int dirb200_grad_clip_coef(const float* grads, int64_t n, float grad_scale, float max_norm, void* workspace,
                           size_t workspace_bytes, float* out, void* stream) {
  DIRB_CHECK_ARG(grads && out && workspace && n > 0 && max_norm > 0.f, "grad_clip_coef: bad arguments");
  DIRB_CHECK_ARG(reinterpret_cast<uintptr_t>(grads) % 16 == 0, "grad_clip_coef: gradient buffer must be 16-byte aligned");
  if (workspace_bytes < dirb200_grad_clip_workspace_bytes()) {
    set_error("grad_clip_coef: workspace too small");
    return DIRB200_ERR_WORKSPACE;
  }
  double* partials = reinterpret_cast<double*>(workspace);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(partials + kClipMaxGrid);
  int grid = grid1d(n / 4 + 1, 256, 4);
  if (grid > kClipMaxGrid) grid = kClipMaxGrid;
  grad_clip_kernel<<<grid, 256, 0, as_stream(stream)>>>(grads, n, grad_scale, max_norm, partials, ticket, out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

size_t dirb200_grad_norm_multi_workspace_bytes(void) { return sizeof(double) * kClipMaxGrid + 16; }

int dirb200_grad_norm_multi(const dirb200_grad_segment* segs_host, int nseg, float max_norm, void* workspace,
                            size_t workspace_bytes, float* out, void* stream) {
  DIRB_CHECK_ARG(segs_host && nseg > 0 && out && workspace && max_norm > 0.f,
                 "grad_norm_multi: bad arguments (segs_host %p, nseg %d, out %p, workspace %p, max_norm %g)",
                 (const void*)segs_host, nseg, (void*)out, workspace, (double)max_norm);
  DIRB_CHECK_ARG(reinterpret_cast<uintptr_t>(workspace) % 8 == 0, "grad_norm_multi: workspace must be 8-byte aligned");
  if (workspace_bytes < dirb200_grad_norm_multi_workspace_bytes()) {
    set_error("grad_norm_multi: workspace too small");
    return DIRB200_ERR_WORKSPACE;
  }
  int64_t total_chunks = 0;
  for (int k = 0; k < nseg; ++k) {
    const dirb200_grad_segment& s = segs_host[k];
    DIRB_CHECK_ARG(s.numel == 0 || s.grad, "grad_norm_multi: segment %d has a null pointer", k);
    DIRB_CHECK_ARG((reinterpret_cast<uintptr_t>(s.grad) & 3) == 0, "grad_norm_multi: segment %d is not 4-byte aligned",
                   k);
    DIRB_CHECK_ARG(s.numel >= 0 && (s.numel - 1) / kAdamChunk < INT32_MAX,
                   "grad_norm_multi: segment %d has numel %lld (0 .. 2^31 chunks of %d)", k, (long long)s.numel,
                   kAdamChunk);
    total_chunks += (s.numel + kAdamChunk - 1) / kAdamChunk;
  }
  // one grid for every launch of the call, so that CTA b of each launch adds into the same partial
  int grid = grid1d(total_chunks, 1, 4);
  if (grid > kClipMaxGrid) grid = kClipMaxGrid;
  double* partials = reinterpret_cast<double*>(workspace);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(partials + kClipMaxGrid);
  GradNormArgs a;
  a.max_norm = max_norm;
  // empty segments are skipped; a launch takes up to kAdamMultiMaxSegs non-empty ones whose chunks fit the int prefix
  int k = 0;
  bool first = true;
  do {
    int ns = 0;
    int64_t chunks = 0;
    a.chunk_start[0] = 0;
    for (; k < nseg && ns < kAdamMultiMaxSegs; ++k) {
      const int64_t c = (segs_host[k].numel + kAdamChunk - 1) / kAdamChunk;
      if (c == 0) continue;
      if (ns > 0 && chunks + c > INT32_MAX) break;
      a.grad[ns] = segs_host[k].grad;
      a.numel[ns] = segs_host[k].numel;
      chunks += c;
      a.chunk_start[++ns] = (int)chunks;
    }
    while (k < nseg && segs_host[k].numel == 0) ++k;     // so that the last launch knows it is the last
    a.nseg = ns;
    a.first = first;
    a.last = k == nseg;
    grad_norm_multi_kernel<<<grid, 256, 0, as_stream(stream)>>>(a, partials, ticket, out);
    DIRB_LAUNCHED();
    first = false;
  } while (k < nseg);
  return DIRB200_OK;
}

}  // extern "C"
