// Bidirectional LSTM layer of sts-b-dir/models.py:40-43 (nn.LSTM(d_word, d_hid, 2, bidirectional=True) behind
// AllenNLP's masked PytorchSeq2SeqWrapper): weight re-layout, the recurrent step (forward and backward, one launch per
// time step, both directions in the same launch) and the bias-gradient reduction.  The time-parallel input projection
// and the weight gradients run on the conv GEMMs (conv_api.cu) as 1x1 convolutions; see imbalanced-regression_b200/rnn.py.
//
// Layouts (Hp = hidden size padded to a multiple of 64, M = rows = 2B, s1 rows then s2 rows, d = direction):
//   gate columns  "interleaved": column n of a direction's 4Hp holds gate (n % 64) / 16 (i, f, g, o) of hidden unit
//                 16 (n / 64) + n % 16, so one 64-wide GEMM-N tile holds all four gates of 16 units and the cell update
//                 runs in that tile's epilogue, each thread owning the four gates of the units it updates.
//   xproj         bf16 [T][M][2][4Hp]   x . W_ih^T in time order (conv_fprop output)
//   whh           bf16 [2][4Hp][Hp]     forward-step B operand (K-major)
//   whhT          bf16 [2][Hp][4Hp]     backward-step B operand (K-major)
//   bias          fp32 [2][4Hp]         b_ih + b_hh
//   h, c          [2][S][M][Hp]         state in STEP order: slot s is step s's input (slot 0 = zeros); S = T + 1 when
//                                       the backward buffers are kept, else 2 (ping-pong).  h bf16, c fp32.
//   gates         fp32 [2][T][M][4Hp]   activated gates of step s (kept for the backward; NULL in inference)
//   y             bf16 [T][M][2Hp]      layer output in time order, direction d at columns [d Hp, d Hp + Hp)
// Step s of the reverse direction processes time tau = len_r - 1 - s of row r, so it starts at each row's own last
// token (pack_padded_sequence semantics).  A row with s >= len_r is inert at step s: it writes zero state, zero
// gradients and a zero output at tau = s.  Every (tau, r, d) output is therefore written exactly once per layer and
// every buffer a weight gradient reads holds zeros outside the mask.
// Invariant: padded weights and biases are zero, so a padded unit has pre-activations 0, i = f = o = 1/2, g = 0 and
// c = h = 0 exactly at every step (c_0 = 0); its gradients are exactly 0 as well.
#include "common.cuh"
#include "tc.cuh"

namespace dirb200 {
namespace {

using namespace tc;
using bf16 = __nv_bfloat16;

constexpr int kStages = 4;
constexpr int kTileBytes = 64 * 128;            // 64 rows x 64 bf16, 128-byte rows
constexpr int kStageBytes = 2 * kTileBytes;     // A tile + B tile
constexpr int kSmemBytes = kStages * kStageBytes + 1024;
constexpr int kMaxT = 4096;
constexpr int kMaxHp = 4096;
constexpr int kMaxM = 65535;

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// One 64 x 64 bf16 K-major tile into shared memory in the wgmma 128-byte-swizzle layout: 16-byte chunk j of row r goes
// to chunk j ^ (r % 8) of the row.  Rows at or beyond `rows` arrive as zeros (cp.async with a 0-byte source).
__device__ __forceinline__ void load_tile(uint32_t dst, const bf16* src, int64_t ld, int rows) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + 128 * i;
    const int r = idx >> 3, j = idx & 7;
    const bool ok = r < rows;
    const bf16* p = ok ? src + r * ld + j * 8 : src;
    cp_async16(dst + r * 128 + ((j ^ (r & 7)) << 4), p, ok ? 16u : 0u);
  }
}

// acc[64 x 64] = A[rows m0.., K] . B[rows n0.., K]^T over K = 64 nk, one warpgroup, a kStages-deep cp.async ring.
// a / b point at the tile's first row; A rows beyond a_rows are read as zeros.
__device__ __forceinline__ void gemm_tile(float (&acc)[32], const bf16* a, int64_t lda, int a_rows, const bf16* b,
                                          int64_t ldb, int nk, uint32_t smem) {
#pragma unroll
  for (int st = 0; st < kStages - 1; ++st) {
    if (st < nk) {
      load_tile(smem + st * kStageBytes, a + st * 64, lda, a_rows);
      load_tile(smem + st * kStageBytes + kTileBytes, b + st * 64, ldb, 64);
    }
    cp_async_commit();
  }
  for (int kb = 0; kb < nk; ++kb) {
    const int pf = kb + kStages - 1;
    if (pf < nk) {
      const uint32_t s = smem + (pf % kStages) * kStageBytes;
      load_tile(s, a + pf * 64, lda, a_rows);
      load_tile(s + kTileBytes, b + pf * 64, ldb, 64);
    }
    cp_async_commit();
    cp_async_wait<kStages - 1>();
    fence_proxy_async();
    __syncthreads();
    const uint32_t s = smem + (kb % kStages) * kStageBytes;
    const uint64_t adesc = make_smem_desc(s, 16u, 1024u);
    const uint64_t bdesc = make_smem_desc(s + kTileBytes, 16u, 1024u);
    wgmma_fence_operands(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_bf16<64, 0, 0>(acc, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(2 * k),
                           (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    __syncthreads();     // every warp is done with this stage before the next iteration refills it
  }
  cp_async_wait<0>();
}

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

struct FwdStep {
  const bf16* xproj;
  const bf16* whh;
  const float* bias;
  const int* lens;
  bf16* h;
  float* c;
  float* gates;
  bf16* y;
  int T, M, Hp, S, s;
};

// grid (4Hp / 64 gate tiles, ceil(M / 64), 2 directions), 128 threads (one warpgroup)
__global__ void __launch_bounds__(128) lstm_fwd_step_kernel(const FwdStep p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int d = blockIdx.z, m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int G = 4 * p.Hp;
  const int sin = p.S == 2 ? (p.s & 1) : p.s, sout = p.S == 2 ? ((p.s + 1) & 1) : p.s + 1;
  const int64_t MH = (int64_t)p.M * p.Hp;
  const bf16* hin = p.h + ((int64_t)d * p.S + sin) * MH;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  if (p.s > 0)     // h_0 = 0: the first step has no recurrent product
    gemm_tile(acc, hin + (int64_t)m0 * p.Hp, p.Hp, p.M - m0, p.whh + ((int64_t)d * G + n0) * p.Hp, p.Hp, p.Hp / 64,
              smem);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fr = lane >> 2, q = lane & 3;
  const float* cin = p.c + ((int64_t)d * p.S + sin) * MH;
  float* cout = p.c + ((int64_t)d * p.S + sout) * MH;
  bf16* hout = p.h + ((int64_t)d * p.S + sout) * MH;
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = m0 + 16 * warp + fr + 8 * rh;
    if (r >= p.M) continue;
    const int len = p.lens[r];
    const bool active = p.s < len;
    const int tau = active ? (d == 0 ? p.s : len - 1 - p.s) : p.s;
    const bf16* xp = p.xproj + (((int64_t)tau * p.M + r) * 2 + d) * G;
    float* gs = p.gates ? p.gates + (((int64_t)d * p.T + p.s) * p.M + r) * G : nullptr;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ul = 8 * hh + 2 * q + e;              // unit within the tile's 16
        const int u = blockIdx.x * 16 + ul;
        float hn = 0.f, cn = 0.f;
        if (active) {
          float a[4];
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int col = n0 + 16 * g + ul;
            a[g] = acc[4 * (2 * g + hh) + 2 * rh + e] + __bfloat162float(xp[col]) + p.bias[d * G + col];
          }
          const float ig = sigm(a[0]), fg = sigm(a[1]), gg = tanhf(a[2]), og = sigm(a[3]);
          cn = fmaf(fg, cin[(int64_t)r * p.Hp + u], ig * gg);
          hn = og * tanhf(cn);
          if (gs) {
            gs[n0 + ul] = ig;
            gs[n0 + 16 + ul] = fg;
            gs[n0 + 32 + ul] = gg;
            gs[n0 + 48 + ul] = og;
          }
        }
        cout[(int64_t)r * p.Hp + u] = cn;
        const bf16 hb = __float2bfloat16_rn(hn);
        hout[(int64_t)r * p.Hp + u] = hb;
        p.y[((int64_t)tau * p.M + r) * 2 * p.Hp + d * p.Hp + u] = hb;
      }
  }
}

struct BwdStep {
  const bf16* whhT;
  const bf16* dy;
  const float* gates;
  const float* c;
  const int* lens;
  float* dc;
  bf16* dg;       // step order [2][T][M][4Hp]
  bf16* dg_time;  // time order [T][M][2][4Hp]
  int T, M, Hp, s;
};

// grid (Hp / 64 unit tiles, ceil(M / 64), 2 directions), 128 threads
__global__ void __launch_bounds__(128) lstm_bwd_step_kernel(const BwdStep p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int d = blockIdx.z, m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int G = 4 * p.Hp;
  const int64_t MH = (int64_t)p.M * p.Hp, MG = (int64_t)p.M * G;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  // dh_s = dgates_{s+1} . W_hh (the last step has no successor)
  if (p.s + 1 < p.T)
    gemm_tile(acc, p.dg + ((int64_t)d * p.T + p.s + 1) * MG + (int64_t)m0 * G, G, p.M - m0,
              p.whhT + ((int64_t)d * p.Hp + n0) * G, G, G / 64, smem);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fr = lane >> 2, q = lane & 3;
  const float* dcin = p.dc + ((int64_t)d * 2 + ((p.s + 1) & 1)) * MH;
  float* dcout = p.dc + ((int64_t)d * 2 + (p.s & 1)) * MH;
  const float* cprev = p.c + ((int64_t)d * (p.T + 1) + p.s) * MH;
  const float* cnew = cprev + MH;
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = m0 + 16 * warp + fr + 8 * rh;
    if (r >= p.M) continue;
    const int len = p.lens[r];
    const bool active = p.s < len;
    const int tau = active ? (d == 0 ? p.s : len - 1 - p.s) : p.s;
    const float* gs = p.gates + (((int64_t)d * p.T + p.s) * p.M + r) * G;
    bf16* dgs = p.dg + (((int64_t)d * p.T + p.s) * p.M + r) * G;
    bf16* dgt = p.dg_time + (((int64_t)tau * p.M + r) * 2 + d) * G;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int u = n0 + 8 * j + 2 * q + e;
        const int gc = (u >> 4) * 64 + (u & 15);        // interleaved column of gate i of unit u
        float da[4] = {0.f, 0.f, 0.f, 0.f}, dcp = 0.f;
        if (active) {
          const float dh = acc[4 * j + 2 * rh + e] + __bfloat162float(p.dy[((int64_t)tau * p.M + r) * 2 * p.Hp + d * p.Hp + u]);
          const float dcn = p.s + 1 < p.T ? dcin[(int64_t)r * p.Hp + u] : 0.f;
          const float ig = gs[gc], fg = gs[gc + 16], gg = gs[gc + 32], og = gs[gc + 48];
          const float tc = tanhf(cnew[(int64_t)r * p.Hp + u]);
          const float dct = dcn + dh * og * (1.f - tc * tc);
          da[0] = dct * gg * ig * (1.f - ig);
          da[1] = dct * cprev[(int64_t)r * p.Hp + u] * fg * (1.f - fg);
          da[2] = dct * ig * (1.f - gg * gg);
          da[3] = dh * tc * og * (1.f - og);
          dcp = dct * fg;
        }
        dcout[(int64_t)r * p.Hp + u] = dcp;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const bf16 v = __float2bfloat16_rn(da[g]);
          dgs[gc + 16 * g] = v;
          dgt[gc + 16 * g] = v;
        }
      }
  }
}

// Interleaved padded column n of one direction -> row of torch's [4H] gate axis (i, f, g, o), or -1 for padding.
__device__ __forceinline__ int gate_row(int n, int H) {
  const int u = (n >> 6) * 16 + (n & 15), g = (n & 63) >> 4;
  return u < H ? g * H + u : -1;
}
// Padded input column j -> torch input index, or -1: the input is `blocks` blocks of `bp` columns, `real` of them used
// (layer 0: one block of d_word; layer k > 0: the two directions' Hp-padded outputs).
__device__ __forceinline__ int in_col(int j, int blocks, int bp, int real) {
  const int b = j / bp, k = j - b * bp;
  return (b < blocks && k < real) ? b * real + k : -1;
}

struct LstmParams {
  const float* w_ih[2];
  const float* w_hh[2];
  const float* b_ih[2];
  const float* b_hh[2];
};

__global__ void lstm_prep_kernel(LstmParams P, int H, int din, int blocks, int bp, int Dp, int Hp, bf16* wih,
                                 bf16* wihT, bf16* whh, bf16* whhT, float* bias) {
  const int G = 4 * Hp;
  const int64_t n_ih = (int64_t)2 * G * Dp, n_hh = (int64_t)2 * G * Hp;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_ih; i += stride) {
    const int j = (int)(i % Dp);
    const int n = (int)(i / Dp);          // [0, 2G): direction n / G
    const int d = n / G, gr = gate_row(n - d * G, H), ic = in_col(j, blocks, bp, H > 0 ? din / blocks : 0);
    const float v = (gr >= 0 && ic >= 0) ? P.w_ih[d][(int64_t)gr * din + ic] : 0.f;
    const bf16 b = __float2bfloat16_rn(v);
    wih[i] = b;
    wihT[(int64_t)j * 2 * G + n] = b;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_hh; i += stride) {
    const int k = (int)(i % Hp);
    const int n = (int)((i / Hp) % G);
    const int d = (int)(i / ((int64_t)Hp * G));
    const int gr = gate_row(n, H);
    const float v = (gr >= 0 && k < H) ? P.w_hh[d][(int64_t)gr * H + k] : 0.f;
    const bf16 b = __float2bfloat16_rn(v);
    whh[i] = b;
    whhT[((int64_t)d * Hp + k) * G + n] = b;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < 2 * G; i += stride) {
    const int d = (int)(i / G), gr = gate_row((int)(i % G), H);
    bias[i] = gr >= 0 ? P.b_ih[d][gr] + P.b_hh[d][gr] : 0.f;
  }
}

struct LstmGrads {
  float* w_ih[2];
  float* w_hh[2];
  float* b_ih[2];
  float* b_hh[2];
};

// Inverse of lstm_prep_kernel for fp32 gradients: one thread per reference-layout element (a gather, every output
// written once).  The bias gradient goes to both b_ih and b_hh.
__global__ void lstm_scatter_kernel(const float* dwih, const float* dwhh, const float* db, int H, int din, int blocks,
                                    int bp, int Dp, int Hp, LstmGrads O) {
  const int G = 4 * Hp;
  const int real = din / blocks;
  const int64_t n_ih = (int64_t)2 * 4 * H * din, n_hh = (int64_t)2 * 4 * H * H;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_ih; i += stride) {
    const int d = (int)(i / ((int64_t)4 * H * din));
    const int64_t k = i - (int64_t)d * 4 * H * din;
    const int gr = (int)(k / din), ic = (int)(k % din);
    const int g = gr / H, u = gr - g * H;
    const int n = (u >> 4) * 64 + g * 16 + (u & 15);
    const int b = ic / real, j = b * bp + (ic - b * real);
    O.w_ih[d][k] = dwih[((int64_t)d * G + n) * Dp + j];
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_hh; i += stride) {
    const int d = (int)(i / ((int64_t)4 * H * H));
    const int64_t k = i - (int64_t)d * 4 * H * H;
    const int gr = (int)(k / H), kk = (int)(k % H);
    const int g = gr / H, u = gr - g * H;
    const int n = (u >> 4) * 64 + g * 16 + (u & 15);
    O.w_hh[d][k] = dwhh[((int64_t)d * G + n) * Hp + kk];
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < 2 * 4 * H; i += stride) {
    const int d = (int)(i / (4 * H)), gr = (int)(i % (4 * H));
    const int g = gr / H, u = gr - g * H;
    const float v = db[d * G + (u >> 4) * 64 + g * 16 + (u & 15)];
    O.b_ih[d][gr] = v;
    O.b_hh[d][gr] = v;
  }
}

// out[col] = sum over rows of x[row][col] (bf16 -> fp32), in a fixed order: block (32 columns x 8 row phases), each
// thread sums its phase's rows in order, then the 8 phases are added in order.  Deterministic, no atomics.
__global__ void __launch_bounds__(256) col_sum_kernel(const bf16* __restrict__ x, int64_t rows, int cols,
                                                      float* __restrict__ out) {
  __shared__ float part[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  float a = 0.f;
  if (col < cols)
    for (int64_t r = threadIdx.y; r < rows; r += 8) a += __bfloat162float(x[r * cols + col]);
  part[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && col < cols) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += part[k][threadIdx.x];
    out[col] = s;
  }
}

int check_dims(int T, int M, int Hp, const char* who) {
  DIRB_CHECK_ARG(T >= 1 && T <= kMaxT, "%s: T must be in [1, %d] (got %d)", who, kMaxT, T);
  DIRB_CHECK_ARG(M >= 1 && M <= kMaxM, "%s: M must be in [1, %d] (got %d)", who, kMaxM, M);
  DIRB_CHECK_ARG(Hp >= 64 && Hp <= kMaxHp && Hp % 64 == 0, "%s: Hp must be a multiple of 64 in [64, %d] (got %d)",
                 who, kMaxHp, Hp);
  return DIRB200_OK;
}

int smem_setup() {
  static bool done = false;
  if (!done) {
    DIRB_CUDA(cudaFuncSetAttribute(lstm_fwd_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    DIRB_CUDA(cudaFuncSetAttribute(lstm_bwd_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    done = true;
  }
  return DIRB200_OK;
}

int fwd_step(const FwdStep& p, cudaStream_t st) {
  if (int rc = smem_setup()) return rc;
  lstm_fwd_step_kernel<<<dim3(4 * p.Hp / 64, (p.M + 63) / 64, 2), 128, kSmemBytes, st>>>(p);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int bwd_step(const BwdStep& p, cudaStream_t st) {
  if (int rc = smem_setup()) return rc;
  lstm_bwd_step_kernel<<<dim3(p.Hp / 64, (p.M + 63) / 64, 2), 128, kSmemBytes, st>>>(p);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // namespace
}  // namespace dirb200

using namespace dirb200;

extern "C" {

int dirb200_lstm_prep_weights(const float* w_ih_f, const float* w_hh_f, const float* b_ih_f, const float* b_hh_f,
                              const float* w_ih_r, const float* w_hh_r, const float* b_ih_r, const float* b_hh_r,
                              int H, int din, int in_blocks, int Hp, int Dp, void* w_ih, void* w_ih_t, void* w_hh,
                              void* w_hh_t, float* bias, void* stream) {
  DIRB_CHECK_ARG(w_ih_f && w_hh_f && b_ih_f && b_hh_f && w_ih_r && w_hh_r && b_ih_r && b_hh_r && w_ih && w_ih_t &&
                     w_hh && w_hh_t && bias,
                 "lstm_prep_weights: null pointer");
  DIRB_CHECK_ARG(H >= 1 && Hp >= H && Hp % 64 == 0 && Hp <= kMaxHp, "lstm_prep_weights: bad H / Hp (%d / %d)", H, Hp);
  DIRB_CHECK_ARG(in_blocks == 1 || in_blocks == 2, "lstm_prep_weights: in_blocks must be 1 or 2");
  DIRB_CHECK_ARG(din >= 1 && din % in_blocks == 0 && Dp % 64 == 0 && Dp % in_blocks == 0 &&
                     din / in_blocks <= Dp / in_blocks && Dp <= 2 * kMaxHp,
                 "lstm_prep_weights: bad input size din %d / Dp %d", din, Dp);
  const LstmParams P{{w_ih_f, w_ih_r}, {w_hh_f, w_hh_r}, {b_ih_f, b_ih_r}, {b_hh_f, b_hh_r}};
  lstm_prep_kernel<<<8 * num_sms(), 256, 0, as_stream(stream)>>>(P, H, din, in_blocks, Dp / in_blocks, Dp, Hp,
                                                                  (bf16*)w_ih, (bf16*)w_ih_t, (bf16*)w_hh,
                                                                  (bf16*)w_hh_t, bias);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_lstm_scatter_grads(const float* dw_ih, const float* dw_hh, const float* db, int H, int din, int in_blocks,
                               int Hp, int Dp, float* gw_ih_f, float* gw_hh_f, float* gb_ih_f, float* gb_hh_f,
                               float* gw_ih_r, float* gw_hh_r, float* gb_ih_r, float* gb_hh_r, void* stream) {
  DIRB_CHECK_ARG(dw_ih && dw_hh && db && gw_ih_f && gw_hh_f && gb_ih_f && gb_hh_f && gw_ih_r && gw_hh_r && gb_ih_r &&
                     gb_hh_r,
                 "lstm_scatter_grads: null pointer");
  DIRB_CHECK_ARG(H >= 1 && Hp >= H && Hp % 64 == 0 && Hp <= kMaxHp, "lstm_scatter_grads: bad H / Hp (%d / %d)", H, Hp);
  DIRB_CHECK_ARG(in_blocks == 1 || in_blocks == 2, "lstm_scatter_grads: in_blocks must be 1 or 2");
  DIRB_CHECK_ARG(din >= 1 && din % in_blocks == 0 && Dp % 64 == 0 && Dp % in_blocks == 0 &&
                     din / in_blocks <= Dp / in_blocks && Dp <= 2 * kMaxHp,
                 "lstm_scatter_grads: bad input size din %d / Dp %d", din, Dp);
  const LstmGrads O{{gw_ih_f, gw_ih_r}, {gw_hh_f, gw_hh_r}, {gb_ih_f, gb_ih_r}, {gb_hh_f, gb_hh_r}};
  lstm_scatter_kernel<<<8 * num_sms(), 256, 0, as_stream(stream)>>>(dw_ih, dw_hh, db, H, din, in_blocks,
                                                                     Dp / in_blocks, Dp, Hp, O);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_lstm_fwd_step(const void* xproj, const void* w_hh, const float* bias, const int* lens, int T, int M,
                          int Hp, int save, int s, void* h, float* c, float* gates, void* y, void* stream) {
  DIRB_CHECK_ARG(xproj && w_hh && bias && lens && h && c && y, "lstm_fwd_step: null pointer");
  DIRB_CHECK_ARG(!save || gates, "lstm_fwd_step: save needs the gates buffer");
  if (int rc = check_dims(T, M, Hp, "lstm_fwd_step")) return rc;
  DIRB_CHECK_ARG(s >= 0 && s < T, "lstm_fwd_step: step %d outside [0, %d)", s, T);
  const FwdStep p{(const bf16*)xproj, (const bf16*)w_hh, bias, lens, (bf16*)h, c, save ? gates : nullptr, (bf16*)y,
                  T, M, Hp, save ? T + 1 : 2, s};
  return fwd_step(p, as_stream(stream));
}

int dirb200_lstm_layer_fwd(const void* xproj, const void* w_hh, const float* bias, const int* lens, int T, int M,
                           int Hp, int save, void* h, float* c, float* gates, void* y, void* stream) {
  DIRB_CHECK_ARG(xproj && w_hh && bias && lens && h && c && y, "lstm_layer_fwd: null pointer");
  DIRB_CHECK_ARG(!save || gates, "lstm_layer_fwd: save needs the gates buffer");
  if (int rc = check_dims(T, M, Hp, "lstm_layer_fwd")) return rc;
  const int S = save ? T + 1 : 2;
  const size_t mh = (size_t)M * Hp;
  cudaStream_t st = as_stream(stream);
  for (int d = 0; d < 2; ++d) {     // slot 0 of each direction: h_0 = c_0 = 0
    DIRB_CUDA(cudaMemsetAsync((bf16*)h + d * S * mh, 0, mh * sizeof(bf16), st));
    DIRB_CUDA(cudaMemsetAsync(c + d * S * mh, 0, mh * sizeof(float), st));
  }
  for (int s = 0; s < T; ++s) {
    const FwdStep p{(const bf16*)xproj, (const bf16*)w_hh, bias, lens, (bf16*)h, c, save ? gates : nullptr,
                    (bf16*)y, T, M, Hp, S, s};
    if (int rc = fwd_step(p, st)) return rc;
  }
  return DIRB200_OK;
}

int dirb200_lstm_bwd_step(const void* w_hh_t, const void* dy, const float* gates, const float* c, const int* lens,
                          int T, int M, int Hp, int s, float* dc, void* dg, void* dg_time, void* stream) {
  DIRB_CHECK_ARG(w_hh_t && dy && gates && c && lens && dc && dg && dg_time, "lstm_bwd_step: null pointer");
  if (int rc = check_dims(T, M, Hp, "lstm_bwd_step")) return rc;
  DIRB_CHECK_ARG(s >= 0 && s < T, "lstm_bwd_step: step %d outside [0, %d)", s, T);
  const BwdStep p{(const bf16*)w_hh_t, (const bf16*)dy, gates, c, lens, dc, (bf16*)dg, (bf16*)dg_time, T, M, Hp, s};
  return bwd_step(p, as_stream(stream));
}

int dirb200_lstm_layer_bwd(const void* w_hh_t, const void* dy, const float* gates, const float* c, const int* lens,
                           int T, int M, int Hp, float* dc, void* dg, void* dg_time, void* stream) {
  DIRB_CHECK_ARG(w_hh_t && dy && gates && c && lens && dc && dg && dg_time, "lstm_layer_bwd: null pointer");
  if (int rc = check_dims(T, M, Hp, "lstm_layer_bwd")) return rc;
  for (int s = T - 1; s >= 0; --s) {
    const BwdStep p{(const bf16*)w_hh_t, (const bf16*)dy, gates, c, lens, dc, (bf16*)dg, (bf16*)dg_time, T, M, Hp, s};
    if (int rc = bwd_step(p, as_stream(stream))) return rc;
  }
  return DIRB200_OK;
}

int dirb200_col_sum_bf16(const void* x, int64_t rows, int cols, float* out, void* stream) {
  DIRB_CHECK_ARG(x && out, "col_sum_bf16: null pointer");
  DIRB_CHECK_ARG(rows >= 1 && cols >= 1, "col_sum_bf16: bad shape");
  col_sum_kernel<<<(cols + 31) / 32, dim3(32, 8), 0, as_stream(stream)>>>((const bf16*)x, rows, cols, out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
