// Evaluation-side reductions of the DIR path (SURVEY §8f-4): overall and many/median/low-shot MSE, L1 and
// geometric-mean error of a prediction vector, in one pass on the device.
//
//   shot_metrics(preds, labels, train_labels, many_shot_thr=100, low_shot_thr=20)   <- agedb-dir/train.py:338-391
//   validate(): overall MSE / L1 / G-Mean                                           <- agedb-dir/train.py:286-335
//   NYUD2 test: align-corners up-sampling + mask + depth metrics per shot group       <- nyud2-dir/test.py:52-55,
//                                                                                      nyud2-dir/util.py:35-133
//
// The reference loops over np.unique(labels) on the host and, per label value l, counts the training samples with
// int(train_label) == l; a test sample therefore belongs to the "many" group when its label's training count is
// > many_thr, to "low" when it is < low_thr (a label value absent from training, or not integer valued, has count
// 0) and to "median" otherwise.  Here: one exact int64 histogram of int(train_label), then one pass over the test
// samples accumulating, per group, (count, sum d^2, sum |d|, sum log|d|) in fp64.
#include "common.cuh"

namespace dirb200 {

// hist[int(label)]++ for 0 <= int(label) < nbins (no clamping, unlike the LDS histogram of datasets.py:60-63)
__global__ void int_label_hist_kernel(const float* __restrict__ labels, int64_t n, int nbins,
                                      unsigned long long* __restrict__ hist) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = labels[i];
    if (!(v == v)) continue;
    const long long b = (long long)v;            // C truncation == numpy astype(int)
    if (b >= 0 && b < nbins) atomicAdd(&hist[b], 1ull);
  }
}

// out[g][k], g = 0 overall, 1 many, 2 median, 3 low; k = 0 count, 1 sum d^2, 2 sum |d|, 3 sum log|d|
__global__ void __launch_bounds__(256)
shot_metrics_kernel(const float* __restrict__ preds, const float* __restrict__ labels, int64_t n,
                    const unsigned long long* __restrict__ train_hist, int nbins, long long many_thr,
                    long long low_thr, double* __restrict__ out) {
  double acc[3][4];
#pragma unroll
  for (int g = 0; g < 3; ++g)
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[g][k] = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float l = labels[i];
    const float df = preds[i] - l;               // float32 difference, as the reference's float32 arrays
    const double d = (double)df;
    long long cnt = 0;                           // training samples whose int(label) equals this label value
    if (l >= 0.f && l < (float)nbins && l == floorf(l)) cnt = (long long)train_hist[(int)l];
    const int g = cnt > many_thr ? 0 : (cnt < low_thr ? 2 : 1);
    const double a = fabs(d);
    const double v[4] = {1.0, d * d, a, log(a)};  // log(0) = -inf -> G-Mean 0, as scipy.stats.gmean
#pragma unroll
    for (int gg = 0; gg < 3; ++gg)
      if (gg == g) {
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[gg][k] += v[k];
      }
  }
  __shared__ double sh[8][12];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int g = 0; g < 3; ++g)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double s = warp_sum(acc[g][k]);
      if (lane == 0) sh[warp][g * 4 + k] = s;
    }
  __syncthreads();
  if (threadIdx.x < 12) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w][threadIdx.x];
    // an empty group contributes exactly 0 (and no -inf from log): skip the atomic when nothing was counted
    const double c = [&] {
      double cc = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) cc += sh[w][(threadIdx.x / 4) * 4];
      return cc;
    }();
    if (c > 0.0) {
      atomicAdd(&out[4 + threadIdx.x], t);       // groups 1..3
      atomicAdd(&out[threadIdx.x & 3], t);       // overall
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// NYUD2-DIR depth evaluation: nyud2-dir/test.py:52-55 (align-corners up-sampling, test mask) + util.py:35-133
// (Evaluator.evaluate / evaluate_shot).  One fused pass per call: the up-sampled prediction is formed in registers
// for the masked pixels only and never stored.  acc[g][k] (g: 0 overall, 1 many, 2 medium, 3 few) is ADDED to:
//   k = 0 NUM (non-NaN targets), 1 sum d^2, 2 sum d, 3 sum d/t, 4 sum |lg10 o - lg10 t|, 5-7 delta1-3 counts,
//   8 NaN targets, 9 +-inf targets.
// Groups 1-3 never hold a NaN or inf target (the reference's int() raises on them), so only their columns 0-7 are
// carried per thread.  Per-CTA fp64 partials go to the workspace and the last CTA sums them in CTA order (the
// loss kernel's ticket pattern): no floating-point atomics, two identical calls give bit-identical sums.
constexpr int kDepthCols = 10;
constexpr int kDepthAcc = 4 * kDepthCols;
constexpr int kDepthMaxGrid = 1024;

struct DepthEvalArgs {
  const float* pred;
  const float* target;
  const uint8_t* mask;
  const uint8_t* group_of_bin;
  int64_t total;     // n_images * h * w
  int ph, pw, h, w, nbins;
  float rheight, rwidth;   // align_corners scales, (float)(in - 1) / (out - 1), as ATen's area_pixel_compute_scale
  bool same;               // (ph, pw) == (h, w): ATen copies instead of interpolating
};

// ATen's upsample_bilinear2d_out_frame (align_corners=True) for one output pixel.  ATen writes
//   h0lambda * (w0lambda * x00 + w1lambda * x01) + h1lambda * (w0lambda * x10 + w1lambda * x11)
// and its sm_90 build contracts every sum into an fma of the FIRST product plus the rounded second one (measured
// against torch's CUDA F.interpolate bit for bit; the other contractions mismatch 30-60 % of the pixels).  The
// contraction is spelled out with intrinsics so that it does not depend on what nvcc chooses here.
__device__ __forceinline__ float upsample_ac_pixel(const float* __restrict__ img, int ph, int pw, float rheight,
                                                   float rwidth, int y, int x) {
  const float h1r = __fmul_rn(rheight, (float)y);
  const int h1 = h1r;
  const int h1p = (h1 < ph - 1) ? 1 : 0;
  const float h1lambda = h1r - h1;
  const float h0lambda = 1.f - h1lambda;
  const float w1r = __fmul_rn(rwidth, (float)x);
  const int w1 = w1r;
  const int w1p = (w1 < pw - 1) ? 1 : 0;
  const float w1lambda = w1r - w1;
  const float w0lambda = 1.f - w1lambda;
  const float* r0 = img + (int64_t)h1 * pw;
  const float* r1 = img + (int64_t)(h1 + h1p) * pw;
  const float top = __fmaf_rn(w0lambda, __ldg(r0 + w1), __fmul_rn(w1lambda, __ldg(r0 + w1 + w1p)));
  const float bot = __fmaf_rn(w0lambda, __ldg(r1 + w1), __fmul_rn(w1lambda, __ldg(r1 + w1 + w1p)));
  return __fmaf_rn(h0lambda, top, __fmul_rn(h1lambda, bot));
}

__global__ void __launch_bounds__(256)
depth_metrics_kernel(DepthEvalArgs a, double* __restrict__ acc_out, double* __restrict__ partials,
                     unsigned int* __restrict__ ticket) {
  double ov[kDepthCols];
  double gr[3][8];
#pragma unroll
  for (int k = 0; k < kDepthCols; ++k) ov[k] = 0.0;
#pragma unroll
  for (int g = 0; g < 3; ++g)
#pragma unroll
    for (int k = 0; k < 8; ++k) gr[g][k] = 0.0;
  const float kLn10 = 2.302585092994046f;       // math.log(10) as the fp32 divisor of lg10, util.py:8-9
  const int64_t hw = (int64_t)a.h * a.w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    if (a.mask && a.mask[i] == 0) continue;     // test.py:54 output[mask]: the taps are loaded for masked pixels only
    const float t = a.target[i];
    if (t != t) {                                // setNanToZero: every term 0, not counted in NUM
      ov[8] += 1.0;
      continue;
    }
    float o;
    if (a.same) {
      o = a.pred[i];
    } else {
      const int64_t img = i / hw;
      const int rem = (int)(i - img * hw);
      const int y = rem / a.w, x = rem - y * a.w;
      o = upsample_ac_pixel(a.pred + img * ((int64_t)a.ph * a.pw), a.ph, a.pw, a.rheight, a.rwidth, y, x);
    }
    const float d = fabsf(o - t);
    const float d2 = d * d;
    const float rel = __fdiv_rn(d, t);
    const float lg = fabsf(__fdiv_rn(logf(o), kLn10) - __fdiv_rn(logf(t), kLn10));
    const float yz = __fdiv_rn(o, t), zy = __fdiv_rn(t, o);
    const float r = (yz < zy) ? zy : yz;         // maxOfTwo: a NaN comparison keeps o / t
    const double v[8] = {1.0, (double)d2, (double)d, (double)rel, (double)lg,
                         r <= 1.25f ? 1.0 : 0.0, r <= 1.5625f ? 1.0 : 0.0, r <= 1.953125f ? 1.0 : 0.0};
#pragma unroll
    for (int k = 0; k < 8; ++k) ov[k] += v[k];
    if (isinf(t)) {                              // int(inf) raises in evaluate_shot: no shot group
      ov[9] += 1.0;
      continue;
    }
    // Evaluator.get_bin_idx: min(int(t * np.float32(10)), 99), the fp32 product truncated toward zero; compared
    // before the conversion so that huge |t| never reaches an out-of-range float -> int cast
    const float p = t * 10.f;
    const int bin = p >= 99.f ? 99 : (p > -1.f ? (int)p : -1);
    const int g = (bin >= 0 && bin < a.nbins) ? (int)__ldg(a.group_of_bin + bin) : 0;
#pragma unroll
    for (int gg = 0; gg < 3; ++gg)
      if (g == gg + 1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) gr[gg][k] += v[k];
      }
  }

  // CTA reduction: warp shuffles, then the 8 warps in order
  __shared__ double sh[8][kDepthAcc];
  __shared__ bool is_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < kDepthCols; ++k) {
    const double s = warp_sum(ov[k]);
    if (lane == 0) sh[warp][k] = s;
  }
#pragma unroll
  for (int g = 0; g < 3; ++g) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const double s = warp_sum(gr[g][k]);
      if (lane == 0) sh[warp][(g + 1) * kDepthCols + k] = s;
    }
    if (lane == 0) sh[warp][(g + 1) * kDepthCols + 8] = sh[warp][(g + 1) * kDepthCols + 9] = 0.0;
  }
  __syncthreads();
  if (threadIdx.x < kDepthAcc) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w][threadIdx.x];
    partials[(int64_t)blockIdx.x * kDepthAcc + threadIdx.x] = t;
    __threadfence();                             // every writer publishes its partial before the ticket is taken
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (gridDim.x == 1) {
      is_last = true;
    } else {
      const unsigned int done = atomicAdd(ticket, 1u);
      is_last = (done == gridDim.x - 1);
    }
  }
  __syncthreads();
  if (is_last && threadIdx.x < kDepthAcc) {
    __threadfence();
    double t = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) t += ((volatile double*)partials)[(int64_t)b * kDepthAcc + threadIdx.x];
    acc_out[threadIdx.x] += t;
  }
}

}  // namespace dirb200

using namespace dirb200;

extern "C" {

int dirb200_int_label_histogram(const float* labels, int64_t n, int nbins, int64_t* hist, void* stream) {
  DIRB_CHECK_ARG(n >= 0 && nbins > 0 && hist && (labels || n == 0), "int_label_histogram: bad arguments");
  if (n == 0) return DIRB200_OK;
  int64_t g = (n + 255) / 256;
  if (g > 4 * num_sms()) g = 4 * num_sms();
  int_label_hist_kernel<<<(unsigned)g, 256, 0, as_stream(stream)>>>(labels, n, nbins,
                                                                  reinterpret_cast<unsigned long long*>(hist));
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_shot_metrics(const float* preds, const float* labels, int64_t n, const int64_t* train_hist, int nbins,
                         int many_shot_thr, int low_shot_thr, double* out16, void* stream) {
  DIRB_CHECK_ARG(n >= 0 && nbins > 0 && train_hist && out16 && ((preds && labels) || n == 0),
                 "shot_metrics: bad arguments");
  DIRB_CHECK_ARG(many_shot_thr >= low_shot_thr, "shot_metrics: many_shot_thr must be >= low_shot_thr");
  cudaStream_t st = as_stream(stream);
  DIRB_CUDA(cudaMemsetAsync(out16, 0, 16 * sizeof(double), st));
  if (n == 0) return DIRB200_OK;
  int64_t g = (n + 255) / 256;
  if (g > 2 * num_sms()) g = 2 * num_sms();
  shot_metrics_kernel<<<(unsigned)g, 256, 0, st>>>(preds, labels, n, reinterpret_cast<const unsigned long long*>(train_hist),
                                                 nbins, many_shot_thr, low_shot_thr, out16);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

static int depth_metrics_grid(int64_t total) {
  int64_t g = (total + 255) / 256;
  const int64_t cap = 2 * (int64_t)num_sms() < kDepthMaxGrid ? 2 * (int64_t)num_sms() : kDepthMaxGrid;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

// [0, 64): ticket; then double partials[grid][4][10]
size_t dirb200_depth_metrics_workspace_bytes(int64_t n_images, int h, int w) {
  if (n_images < 0 || h <= 0 || w <= 0) return 0;
  return 64 + sizeof(double) * kDepthAcc * (size_t)depth_metrics_grid(n_images * h * w);
}

int dirb200_depth_metrics_accumulate(const float* pred, int ph, int pw, const float* target, const uint8_t* mask,
                                     int64_t n_images, int h, int w, const uint8_t* group_of_bin, int nbins,
                                     double* acc, void* workspace, size_t workspace_bytes, void* stream) {
  DIRB_CHECK_ARG(n_images >= 0 && h > 0 && w > 0 && ph > 0 && pw > 0, "depth_metrics: bad shape");
  DIRB_CHECK_ARG((int64_t)h * w < (1ll << 31) && (int64_t)ph * pw < (1ll << 31),
                 "depth_metrics: an image must have fewer than 2^31 pixels");
  DIRB_CHECK_ARG(nbins >= 0 && (nbins == 0) == (group_of_bin == nullptr),
                 "depth_metrics: group_of_bin must be given exactly when nbins > 0");
  DIRB_CHECK_ARG(acc && workspace && ((pred && target) || n_images == 0), "depth_metrics: null pointer");
  if (workspace_bytes < dirb200_depth_metrics_workspace_bytes(n_images, h, w)) {
    set_error("depth_metrics: workspace too small");
    return DIRB200_ERR_WORKSPACE;
  }
  const int64_t total = n_images * h * w;
  if (total == 0) return DIRB200_OK;
  DepthEvalArgs a;
  a.pred = pred;
  a.target = target;
  a.mask = mask;
  a.group_of_bin = group_of_bin;
  a.total = total;
  a.ph = ph;
  a.pw = pw;
  a.h = h;
  a.w = w;
  a.nbins = nbins;
  // area_pixel_compute_scale(align_corners=True): fp32 quotient, 0 for a single output row / column
  a.rheight = h > 1 ? (float)(ph - 1) / (float)(h - 1) : 0.f;
  a.rwidth = w > 1 ? (float)(pw - 1) / (float)(w - 1) : 0.f;
  a.same = (ph == h && pw == w);
  const int grid = depth_metrics_grid(total);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
  double* partials = reinterpret_cast<double*>(static_cast<char*>(workspace) + 64);
  cudaStream_t st = as_stream(stream);
  if (grid > 1) DIRB_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
  depth_metrics_kernel<<<grid, 256, 0, st>>>(a, acc, partials, ticket);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
