// The non-recurrent parts of sts-b-dir/models.py's HeadlessPairEncoder (models.py:137-166): the embedding lookup with
// its dropout into the padded bf16 input of the first LSTM layer, and the masked max over time with the pair features
// [u, v, |u - v|, u * v].  Rows are M = 2B: the B s1 sentences, then the B s2 sentences.  Dropout arrives as an fp32
// multiplier (keep / (1 - p), or 0) per element, drawn by the caller; NULL means no dropout.
#include "common.cuh"

namespace dirb200 {
namespace {

using bf16 = __nv_bfloat16;

// x[t][m][j] = emb[ids[m][t]][j] * dmul[m][t][j] for t < lens[m] and j < D, else 0 (the positions outside the mask
// feed the first layer's weight gradient and must be zeros).  An id outside [0, V) gives NaN.
__global__ void embed_gather_kernel(const int64_t* __restrict__ ids, const int* __restrict__ lens,
                                    const float* __restrict__ emb, const float* __restrict__ dmul, int64_t V, int M,
                                    int T, int D, int Dp, bf16* __restrict__ x) {
  const int64_t total = (int64_t)T * M * Dp;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % Dp);
    const int64_t tm = i / Dp;
    const int m = (int)(tm % M), t = (int)(tm / M);
    float v = 0.f;
    if (j < D && t < lens[m]) {
      const int64_t id = ids[(int64_t)m * T + t];
      v = (id >= 0 && id < V) ? emb[id * D + j] : __int_as_float(0x7fc00000);
      if (dmul) v *= dmul[((int64_t)m * T + t) * D + j];
    }
    x[i] = __float2bfloat16_rn(v);
  }
}

// dW[id] = sum over the unmasked positions p holding id, in position order p = m T + t, of dx[t][m][:] * dmul.  One
// block per position; only the first position of each id (its "leader") does the sum, so every row is written by one
// block and the order is fixed: deterministic without atomics.  Rows of ids that do not occur are zeroed beforehand;
// so is the padding row (F.embedding's padding_idx: no gradient) and ids outside [0, V) contribute nothing.
// Cost: each leader scans the positions once per 128 columns, O(P x distinct ids) id compares.
__global__ void __launch_bounds__(128) embed_grad_kernel(const int64_t* __restrict__ ids, const int* __restrict__ lens,
                                                         const bf16* __restrict__ dx, const float* __restrict__ dmul,
                                                         int M, int T, int D, int Dp, int64_t V, int64_t pad,
                                                         float* __restrict__ dw) {
  const int p = blockIdx.x;
  const int m = p / T, t = p - m * T;
  if (t >= lens[m]) return;
  const int64_t id = ids[p];
  if (id < 0 || id >= V || id == pad) return;
  int earlier = 0;
  for (int q = threadIdx.x; q < p; q += blockDim.x) {
    const int mq = q / T;
    if (q - mq * T < lens[mq] && ids[q] == id) earlier = 1;
  }
  if (__syncthreads_or(earlier)) return;
  const int P = M * T;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    float acc = 0.f;
    for (int q = p; q < P; ++q) {
      const int mq = q / T, tq = q - mq * T;
      if (tq >= lens[mq] || ids[q] != id) continue;
      float g = __bfloat162float(dx[((int64_t)tq * M + mq) * Dp + j]);
      if (dmul) g *= dmul[(int64_t)q * D + j];
      acc += g;
    }
    dw[id * D + j] = acc;
  }
}

// One thread per (b, j), j < 2H the column of the reference's [B, 2H] encoder output (direction j / H, unit j % H):
// u = max_{t < len} y[t][b] * dmul, v the same for row B + b.  Ties go to the first maximal t.
__global__ void pair_maxpool_fwd_kernel(const bf16* __restrict__ y, const int* __restrict__ lens,
                                        const float* __restrict__ dmul, int B, int T, int H, int Hp,
                                        float* __restrict__ feat, int* __restrict__ arg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int H2 = 2 * H;
  if (i >= B * H2) return;
  const int b = i / H2, j = i - b * H2;
  const int col = (j / H) * Hp + (j % H);
  const int M = 2 * B;
  float uv[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int r = b + k * B;
    float best = -INFINITY;
    int bt = 0;
    for (int t = 0; t < lens[r]; ++t) {
      float v = __bfloat162float(y[((int64_t)t * M + r) * 2 * Hp + col]);
      if (dmul) v *= dmul[((int64_t)r * T + t) * H2 + j];
      if (v > best) { best = v; bt = t; }
    }
    uv[k] = best;
    arg[(int64_t)r * H2 + j] = bt;
  }
  float* f = feat + (int64_t)b * 4 * H2;
  f[j] = uv[0];
  f[H2 + j] = uv[1];
  f[2 * H2 + j] = fabsf(uv[0] - uv[1]);
  f[3 * H2 + j] = uv[0] * uv[1];
}

// dy (zeroed by the caller) at the argmax time of each (row, column): du = g0 + sign(u - v) g2 + v g3 and
// dv = g1 - sign(u - v) g2 + u g3 (sign 0 at u == v, as torch's abs backward), times the dropout multiplier.
__global__ void pair_maxpool_bwd_kernel(const float* __restrict__ gfeat, const float* __restrict__ feat,
                                        const int* __restrict__ arg, const float* __restrict__ dmul, int B, int T,
                                        int H, int Hp, bf16* __restrict__ dy) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int H2 = 2 * H;
  if (i >= B * H2) return;
  const int b = i / H2, j = i - b * H2;
  const int col = (j / H) * Hp + (j % H);
  const int M = 2 * B;
  const float* g = gfeat + (int64_t)b * 4 * H2;
  const float u = feat[(int64_t)b * 4 * H2 + j], v = feat[(int64_t)b * 4 * H2 + H2 + j];
  const float sg = (u > v) ? 1.f : (u < v ? -1.f : 0.f);
  const float d[2] = {g[j] + sg * g[2 * H2 + j] + v * g[3 * H2 + j], g[H2 + j] - sg * g[2 * H2 + j] + u * g[3 * H2 + j]};
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int r = b + k * B;
    const int t = arg[(int64_t)r * H2 + j];
    float x = d[k];
    if (dmul) x *= dmul[((int64_t)r * T + t) * H2 + j];
    dy[((int64_t)t * M + r) * 2 * Hp + col] = __float2bfloat16_rn(x);
  }
}

constexpr int kMaxT = 4096;

int check(int M, int T, const char* who) {
  DIRB_CHECK_ARG(M >= 1 && M <= 65535, "%s: rows must be in [1, 65535] (got %d)", who, M);
  DIRB_CHECK_ARG(T >= 1 && T <= kMaxT, "%s: T must be in [1, %d] (got %d)", who, kMaxT, T);
  return DIRB200_OK;
}

}  // namespace
}  // namespace dirb200

using namespace dirb200;

extern "C" {

int dirb200_embed_gather(const int64_t* ids, const int* lens, const float* emb, const float* dmul, int64_t V, int M,
                         int T, int D, int Dp, void* x, void* stream) {
  DIRB_CHECK_ARG(ids && lens && emb && x, "embed_gather: null pointer");
  if (int rc = check(M, T, "embed_gather")) return rc;
  DIRB_CHECK_ARG(V >= 1 && D >= 1 && Dp >= D && Dp % 64 == 0, "embed_gather: bad V %lld / D %d / Dp %d", (long long)V,
                 D, Dp);
  const int64_t total = (int64_t)T * M * Dp;
  const int64_t grid = (total + 255) / 256;
  embed_gather_kernel<<<(unsigned)(grid < 8 * num_sms() ? grid : 8 * num_sms()), 256, 0, as_stream(stream)>>>(
      ids, lens, emb, dmul, V, M, T, D, Dp, (bf16*)x);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_embed_grad(const int64_t* ids, const int* lens, const void* dx, const float* dmul, int64_t V, int M, int T,
                       int D, int Dp, int64_t padding_index, float* dw, void* stream) {
  DIRB_CHECK_ARG(ids && lens && dx && dw, "embed_grad: null pointer");
  if (int rc = check(M, T, "embed_grad")) return rc;
  DIRB_CHECK_ARG(V >= 1 && D >= 1 && Dp >= D && Dp % 64 == 0, "embed_grad: bad V %lld / D %d / Dp %d", (long long)V, D,
                 Dp);
  DIRB_CHECK_ARG((int64_t)M * T < (1LL << 31), "embed_grad: too many positions");
  cudaStream_t st = as_stream(stream);
  DIRB_CUDA(cudaMemsetAsync(dw, 0, (size_t)V * D * sizeof(float), st));
  embed_grad_kernel<<<M * T, 128, 0, st>>>(ids, lens, (const bf16*)dx, dmul, M, T, D, Dp, V,
                                                padding_index, dw);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_pair_maxpool_fwd(const void* y, const int* lens, const float* dmul, int B, int T, int H, int Hp,
                             float* feat, int* arg, void* stream) {
  DIRB_CHECK_ARG(y && lens && feat && arg, "pair_maxpool_fwd: null pointer");
  if (int rc = check(2 * B, T, "pair_maxpool_fwd")) return rc;
  DIRB_CHECK_ARG(H >= 1 && Hp >= H, "pair_maxpool_fwd: bad H %d / Hp %d", H, Hp);
  const int n = B * 2 * H;
  pair_maxpool_fwd_kernel<<<(n + 255) / 256, 256, 0, as_stream(stream)>>>((const bf16*)y, lens, dmul, B, T, H, Hp,
                                                                          feat, arg);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_pair_maxpool_bwd(const float* gfeat, const float* feat, const int* arg, const float* dmul, int B, int T,
                             int H, int Hp, void* dy, void* stream) {
  DIRB_CHECK_ARG(gfeat && feat && arg && dy, "pair_maxpool_bwd: null pointer");
  if (int rc = check(2 * B, T, "pair_maxpool_bwd")) return rc;
  DIRB_CHECK_ARG(H >= 1 && Hp >= H, "pair_maxpool_bwd: bad H %d / Hp %d", H, Hp);
  cudaStream_t st = as_stream(stream);
  DIRB_CUDA(cudaMemsetAsync(dy, 0, (size_t)T * 2 * B * 2 * Hp * sizeof(bf16), st));
  const int n = B * 2 * H;
  pair_maxpool_bwd_kernel<<<(n + 255) / 256, 256, 0, st>>>(gfeat, feat, arg, dmul, B, T, H, Hp, (bf16*)dy);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
