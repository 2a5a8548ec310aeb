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
#include "bins.cuh"

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

// out[g][k], g = 0 overall, 1 many, 2 median, 3 low; k = 0 count, 1 sum d^2, 2 sum |d|, 3 sum log|d|.
// One CTA: every sum has a fixed order (a grid-stride loop per thread, warp shuffles, the warps in order, overall =
// many + median + low), so two identical calls give identical bits.  It runs once per validation pass over at most
// a few ten thousand samples.
constexpr int kShotThreads = 512;

__global__ void __launch_bounds__(kShotThreads)
shot_metrics_kernel(const float* __restrict__ preds, const float* __restrict__ labels, int64_t n,
                    const unsigned long long* __restrict__ train_hist, int nbins, long long many_thr,
                    long long low_thr, double* __restrict__ out) {
  double acc[3][4];
#pragma unroll
  for (int g = 0; g < 3; ++g)
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[g][k] = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
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
  __shared__ double sh[kShotThreads / 32][12];
  __shared__ double tot[12];
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
    tot[threadIdx.x] = t;
    out[4 + threadIdx.x] = t;                    // groups 1..3
  }
  __syncthreads();
  // an empty group holds exact zeros (no log was added), so it leaves the overall sums unchanged
  if (threadIdx.x < 4) out[threadIdx.x] = (tot[threadIdx.x] + tot[4 + threadIdx.x]) + tot[8 + threadIdx.x];
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

// ------------------------------------------------------------------------------------------------------------------
// STS-B-DIR's STSShotAverage.get_metric (sts-b-dir/util.py:101-172): count, MSE, L1, G-mean, Pearson and Spearman over
// x = 5 pred (fp64) and y = label, overall and per many / medium / few group.  A label's group is its bin under the
// DIRB200_BIN_EDGES5 rule with 50 bins (util.py:115-120: np.histogram edges over [0, 5], 5.0 in the last bin) looked
// up in util.py:110-113's table.  A negative label, whose reference bin is -1, is in no list and so counts as few.
//
// Spearman is Pearson of the average ranks within each group (scipy's rankdata('average')).  stsb_rank_kernel gets
// them as exact counts, 2 rank = #less + #less-or-equal + 1, from a tiled O(N^2) comparison of every pair: no sort, no
// floating point.  The order of fp32 preds is the order of 5 pred in fp64 (exact), so the raw fp32 values are
// compared.  stsb_metrics_kernel is one CTA: a first pass of sums, then centred sums about the means of the first, and
// the final formulas; every sum has a fixed order, so two identical calls give identical bits.
constexpr int kStsbGroups = 4;   // 0 overall, 1 many, 2 medium, 3 few (the order of util.py:143)
constexpr int kStsbOut = 6;      // num_samples, mse, l1, gmean, pearsonr, spearmanr
constexpr int64_t kStsbMaxN = 1ll << 22;

__constant__ unsigned char kStsbShotOfBin[50] = {
    // util.py:110-113, bins 0 .. 49
    1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 1, 3, 1, 3, 1, 3, 1, 3, 1, 3, 1, 3, 1, 3, 1,
    3, 1, 2, 1, 3, 1, 3, 1, 3, 1, 2, 1, 2, 1, 3, 1, 3, 1, 3, 1, 3, 1, 3, 1, 1};

__device__ __forceinline__ int stsb_group(float label) {
  if (!(label >= 0.f)) return 3;     // bin -1 (a NaN label is out of the reference's contract: few as well)
  return kStsbShotOfBin[bin_of(DIRB200_BIN_EDGES5, label, 0.f, 49.f, 50, false, false)];
}

// r2[i] = twice the average rank of pred_i and label_i, overall (.x, .y) and within i's group (.z, .w)
__global__ void __launch_bounds__(256)
stsb_rank_kernel(const float* __restrict__ preds, const float* __restrict__ labels, int n, int4* __restrict__ r2) {
  __shared__ float sp[256], sl[256];
  __shared__ int sg[256];
  const int i = blockIdx.x * 256 + threadIdx.x;
  const bool in = i < n;
  const float p = in ? preds[i] : 0.f, l = in ? labels[i] : 0.f;
  const int g = in ? stsb_group(l) : 0;
  int ap = 0, al = 0, gp = 0, gl = 0;    // #less + #less-or-equal, overall and in the group
  for (int j0 = 0; j0 < n; j0 += 256) {
    __syncthreads();
    const int j = j0 + threadIdx.x;
    if (j < n) {
      sp[threadIdx.x] = preds[j];
      sl[threadIdx.x] = labels[j];
      sg[threadIdx.x] = stsb_group(labels[j]);
    }
    __syncthreads();
    const int m = n - j0 < 256 ? n - j0 : 256;
#pragma unroll 4
    for (int k = 0; k < m; ++k) {
      const float q = sp[k], r = sl[k];
      const int cp = (q < p) + (q <= p), cl = (r < l) + (r <= l);
      ap += cp;
      al += cl;
      if (sg[k] == g) {
        gp += cp;
        gl += cl;
      }
    }
  }
  if (in) r2[i] = make_int4(ap + 1, al + 1, gp + 1, gl + 1);
}

// per-thread sums: [group][quantity]; a sample adds to group 0 and to its own group
template <int K>
__device__ __forceinline__ void stsb_add(double (&acc)[kStsbGroups][K], int g, const double (&v0)[K],
                                         const double (&vg)[K]) {
#pragma unroll
  for (int k = 0; k < K; ++k) acc[0][k] += v0[k];
#pragma unroll
  for (int gg = 1; gg < kStsbGroups; ++gg)
    if (gg == g) {
#pragma unroll
      for (int k = 0; k < K; ++k) acc[gg][k] += vg[k];
    }
}

// sums acc over the CTA (warp shuffles, then the warps in order) into tot, visible to every thread on return
template <int K>
__device__ void stsb_cta_sum(double (&acc)[kStsbGroups][K], double* sh, double* tot) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll
  for (int g = 0; g < kStsbGroups; ++g)
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double s = warp_sum(acc[g][k]);
      if (lane == 0) sh[warp * kStsbGroups * K + g * K + k] = s;
    }
  __syncthreads();
  if (threadIdx.x < kStsbGroups * K) {
    double t = 0.0;
    for (int w = 0; w < nw; ++w) t += sh[w * kStsbGroups * K + threadIdx.x];
    tot[threadIdx.x] = t;
  }
  __syncthreads();
}

__device__ __forceinline__ double stsb_clip_corr(double r) { return r > 1.0 ? 1.0 : (r < -1.0 ? -1.0 : r); }

// rank of a sample from r2 (NaN for a NaN value: scipy's rankdata propagates it)
__device__ __forceinline__ double stsb_rank(int twice, float v) { return v == v ? 0.5 * (double)twice : (double)NAN; }

constexpr int kStsbSum1 = 8;   // n, sum x, sum y, sum rx, sum ry, sum d^2, sum |d|, sum log |d|'
constexpr int kStsbSum2 = 8;   // Sxx, Syy, Sxy, Srxrx, Sryry, Srxry, #(x not at the constant rank), same for y

__global__ void __launch_bounds__(256)
stsb_metrics_kernel(const float* __restrict__ preds, const float* __restrict__ labels, int n,
                    const int4* __restrict__ r2, double* __restrict__ out) {
  __shared__ double sh[8 * kStsbGroups * kStsbSum1];
  __shared__ double s1[kStsbGroups * kStsbSum1], s2[kStsbGroups * kStsbSum2];
  double acc[kStsbGroups][kStsbSum1];
#pragma unroll
  for (int g = 0; g < kStsbGroups; ++g)
#pragma unroll
    for (int k = 0; k < kStsbSum1; ++k) acc[g][k] = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float p = preds[i], l = labels[i];
    const int4 r = r2[i];
    const double x = (double)p * 5.0, y = (double)l;
    const double d = x - y, a = fabs(d);
    const double lg = log(a == 0.0 ? 1e-10 : a);      // util.py:152-154: an exact zero difference counts as 1e-10
    const double v0[kStsbSum1] = {1.0, x, y, stsb_rank(r.x, p), stsb_rank(r.y, l), d * d, a, lg};
    const double vg[kStsbSum1] = {1.0, x, y, stsb_rank(r.z, p), stsb_rank(r.w, l), d * d, a, lg};
    stsb_add(acc, stsb_group(l), v0, vg);
  }
  stsb_cta_sum(acc, sh, s1);

  double acc2[kStsbGroups][kStsbSum2];
#pragma unroll
  for (int g = 0; g < kStsbGroups; ++g)
#pragma unroll
    for (int k = 0; k < kStsbSum2; ++k) acc2[g][k] = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float p = preds[i], l = labels[i];
    const int4 r = r2[i];
    const int g = stsb_group(l);
    const double x = (double)p * 5.0, y = (double)l;
    double v[2][kStsbSum2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int gg = s == 0 ? 0 : g;
      const double* m = s1 + gg * kStsbSum1;
      const double cnt = m[0];
      const double xm = x - m[1] / cnt, ym = y - m[2] / cnt;
      const double rx = stsb_rank(s == 0 ? r.x : r.z, p) - m[3] / cnt;
      const double ry = stsb_rank(s == 0 ? r.y : r.w, l) - m[4] / cnt;
      // a group's x is constant exactly when every member's twice-rank is cnt + 1 (all tied)
      const int tx = s == 0 ? r.x : r.z, ty = s == 0 ? r.y : r.w;
      v[s][0] = xm * xm;
      v[s][1] = ym * ym;
      v[s][2] = xm * ym;
      v[s][3] = rx * rx;
      v[s][4] = ry * ry;
      v[s][5] = rx * ry;
      v[s][6] = (double)tx != cnt + 1.0 ? 1.0 : 0.0;
      v[s][7] = (double)ty != cnt + 1.0 ? 1.0 : 0.0;
    }
    stsb_add(acc2, g, v[0], v[1]);
  }
  stsb_cta_sum(acc2, sh, s2);

  if (threadIdx.x < kStsbGroups) {
    const int g = threadIdx.x;
    const double* a = s1 + g * kStsbSum1;
    const double* b = s2 + g * kStsbSum2;
    const double cnt = a[0];
    double* o = out + g * kStsbOut;
    o[0] = cnt;
    if (cnt == 0.0) {                      // util.py: an empty group reports 0 for every metric
      o[1] = o[2] = o[3] = o[4] = o[5] = 0.0;
      return;
    }
    o[1] = a[5] / cnt;
    o[2] = a[6] / cnt;
    o[3] = exp(a[7] / cnt);                // scipy.stats.gmean: exp(mean(log))
    if (cnt < 2.0) {                       // util.py:161, 163: size 1 reports 0
      o[4] = o[5] = 0.0;
      return;
    }
    // scipy.stats.pearsonr: NaN for a constant input, the centred formula clipped to [-1, 1], rounded for n == 2
    double pr = stsb_clip_corr(b[2] / (sqrt(b[0]) * sqrt(b[1])));
    if (cnt == 2.0) pr = rint(pr);
    if (b[6] == 0.0 || b[7] == 0.0) pr = (double)NAN;
    o[4] = pr;
    // scipy.stats.spearmanr: np.corrcoef of the ranks (all-tied ranks give 0 / 0 = NaN)
    o[5] = stsb_clip_corr(b[5] / (sqrt(b[3]) * sqrt(b[4])));
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
  if (n == 0) {
    DIRB_CUDA(cudaMemsetAsync(out16, 0, 16 * sizeof(double), st));
    return DIRB200_OK;
  }
  shot_metrics_kernel<<<1, kShotThreads, 0, st>>>(preds, labels, n, reinterpret_cast<const unsigned long long*>(train_hist),
                                                 nbins, many_shot_thr, low_shot_thr, out16);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

size_t dirb200_stsb_shot_metrics_workspace_bytes(int64_t n) { return n > 0 ? sizeof(int4) * (size_t)n : 0; }

int dirb200_stsb_shot_metrics(const float* preds, const float* labels, int64_t n, void* workspace,
                              size_t workspace_bytes, double* out24, void* stream) {
  // the rank counts reach 2 n + 1 in int32, and the pair comparison is quadratic: 2^22 keeps both bounded
  DIRB_CHECK_ARG(n >= 0 && n <= kStsbMaxN, "stsb_shot_metrics: n %lld out of range (0 .. 2^22)", (long long)n);
  DIRB_CHECK_ARG(out24 && (n == 0 || (preds && labels && workspace)), "stsb_shot_metrics: null pointer");
  DIRB_CHECK_ARG(reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "stsb_shot_metrics: workspace must be 16-byte aligned");
  if (workspace_bytes < dirb200_stsb_shot_metrics_workspace_bytes(n)) {
    set_error("stsb_shot_metrics: workspace too small");
    return DIRB200_ERR_WORKSPACE;
  }
  cudaStream_t st = as_stream(stream);
  int4* r2 = reinterpret_cast<int4*>(workspace);
  if (n > 0) {
    stsb_rank_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(preds, labels, (int)n, r2);
    DIRB_LAUNCHED();
  }
  stsb_metrics_kernel<<<1, 256, 0, st>>>(preds, labels, (int)n, r2, out24);
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
