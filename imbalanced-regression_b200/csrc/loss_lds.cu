// Stage (iii): weighted regression losses (fused forward + backward) and LDS
// label-distribution-smoothing weights.
//
//   weighted_{mse,l1,focal_mse,focal_l1,huber}_loss  <- agedb-dir/loss.py:5-48
//   label histogram / re-weighting / LDS convolve     <- agedb-dir/datasets.py:55-83
#include "common.cuh"

namespace dirb200 {

struct LossParams {
  int kind, activate;
  float beta, gamma, grad_scale;
};

__device__ __forceinline__ void loss_elem(const LossParams& p, float x, float t, float w, float& l, float& g) {
  const float d = x - t;
  const float a = fabsf(d);
  const float sg = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
  switch (p.kind) {
    case DIRB200_LOSS_MSE:
      l = d * d;
      g = 2.f * d;
      break;
    case DIRB200_LOSS_L1:
      l = a;
      g = sg;
      break;
    case DIRB200_LOSS_HUBER: {
      const bool small = a < p.beta;
      l = small ? 0.5f * a * a / p.beta : a - 0.5f * p.beta;
      g = small ? d / p.beta : sg;
      break;
    }
    default: {  // focal_mse / focal_l1
      float fb, dfb;
      if (p.activate == DIRB200_ACT_TANH) {
        fb = tanhf(p.beta * a);
        dfb = p.beta * (1.f - fb * fb);
      } else {
        const float s = 1.f / (1.f + expf(-p.beta * a));
        fb = 2.f * s - 1.f;
        dfb = 2.f * p.beta * s * (1.f - s);
      }
      float f, df;
      if (p.gamma == 1.f) {
        f = fb;
        df = dfb;
      } else {
        f = powf(fb, p.gamma);
        df = p.gamma * powf(fb, p.gamma - 1.f) * dfb;
      }
      if (p.kind == DIRB200_LOSS_FOCAL_MSE) {
        l = d * d * f;
        g = 2.f * d * f + d * d * df * sg;
      } else {
        l = a * f;
        g = sg * f + a * df * sg;
      }
      break;
    }
  }
  l *= w;
  g *= w;
}

// partials[grid] doubles + ticket (uint32) live in the workspace.
__global__ void __launch_bounds__(256)
loss_fwd_bwd_kernel(LossParams p, const float* __restrict__ pred, const float* __restrict__ target,
                    const float* __restrict__ weight, int64_t n, float* __restrict__ loss_out,
                    float* __restrict__ grad_out, double* __restrict__ partials, unsigned int* __restrict__ ticket) {
  __shared__ double sh[8];
  __shared__ bool is_last;
  const float inv_n = 1.f / (float)n;
  double acc = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float l, g;
    loss_elem(p, pred[i], target[i], weight ? weight[i] : 1.f, l, g);
    acc += (double)l;
    if (grad_out) grad_out[i] = g * inv_n * p.grad_scale;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += sh[w];
    partials[blockIdx.x] = t;
    if (gridDim.x == 1) {
      is_last = true;
    } else {
      __threadfence();
      const unsigned int done = atomicAdd(ticket, 1u);
      is_last = (done == gridDim.x - 1);
    }
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    double t = 0.0;
    for (int i = threadIdx.x; i < gridDim.x; i += blockDim.x) t += ((volatile double*)partials)[i];
    t = warp_sum(t);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int w = 0; w < (blockDim.x >> 5); ++w) s += sh[w];
      loss_out[0] = (float)(s / (double)n);
    }
  }
}

// ---------------------------------------------------------------------- LDS
__global__ void lds_hist_kernel(const float* __restrict__ labels, int64_t n, int max_target,
                                unsigned long long* __restrict__ hist) {
  extern __shared__ unsigned int shh[];
  for (int i = threadIdx.x; i < max_target; i += blockDim.x) shh[i] = 0u;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)labels[i];                 // int(label): truncation toward zero
    b = max(0, min(max_target - 1, b));     // min(max_target-1, .); negatives are a contract violation -> bin 0
    atomicAdd(&shh[b], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < max_target; i += blockDim.x)
    if (shh[i]) atomicAdd(&hist[i], (unsigned long long)shh[i]);
}

struct LdsWindow {
  double w[33];
};

// single block: per-bin value -> inverse (as float32) -> scaling.  scratch layout:
// val[max_target] | inv[max_target] (float32 value stored as double) | scaling
__global__ void lds_bins_kernel(const long long* __restrict__ hist, int max_target, int reweight, LdsWindow win,
                                int ks, int64_t n, double* __restrict__ scratch) {
  double* val = scratch;
  double* inv = scratch + max_target;
  double* scaling = scratch + 2 * max_target;
  for (int i = threadIdx.x; i < max_target; i += blockDim.x) {
    const double h = (double)hist[i];
    val[i] = (reweight == DIRB200_REWEIGHT_SQRT_INV) ? sqrt(h) : fmin(fmax(h, 5.0), 1000.0);
  }
  __syncthreads();
  if (ks > 0) {
    const int hk = ks / 2;
    for (int i = threadIdx.x; i < max_target; i += blockDim.x) {
      // scipy.ndimage.convolve1d symmetric path: centre tap, then outer pairs inwards; no FMA
      double acc = __dmul_rn(val[i], win.w[hk]);
      for (int j = -hk; j < 0; ++j) {
        const int a = i + j, b = i - j;
        const double xa = (a >= 0) ? val[a] : 0.0;
        const double xb = (b < max_target) ? val[b] : 0.0;
        acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(xa, xb), win.w[hk + j]));
      }
      // output takes the input dtype: int64 histogram on the 'inverse' path -> truncation
      inv[i] = (reweight == DIRB200_REWEIGHT_INVERSE) ? trunc(acc) : acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < max_target; i += blockDim.x) val[i] = inv[i];
    __syncthreads();
  }
  for (int i = threadIdx.x; i < max_target; i += blockDim.x)
    inv[i] = (hist[i] > 0) ? (double)(float)(1.0 / val[i]) : 0.0;   // np.float32(1 / x)
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < max_target; ++i) s += (double)hist[i] * inv[i];
    // scaling = len / sum(w): float32 in the reference
    scaling[0] = (double)((float)n / (float)s);
  }
}

__global__ void lds_gather_kernel(const float* __restrict__ labels, int64_t n, int max_target,
                                  const double* __restrict__ scratch, float* __restrict__ out) {
  const double* inv = scratch + max_target;
  const float scaling = (float)scratch[2 * max_target];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)labels[i];
    b = max(0, min(max_target - 1, b));
    out[i] = __fmul_rn(scaling, (float)inv[b]);
  }
}

// out[i] = table[min(int(values[i] * mult), max_bin)]   (per-pixel LDS weight lookup, nyud2-dir/loaddata.py:55-64)
__global__ void lds_table_lookup_kernel(const float* __restrict__ values, int64_t n, float mult, int max_bin,
                                        const float* __restrict__ table, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)__fmul_rn(values[i], mult);
    b = max(0, min(max_bin, b));
    out[i] = table[b];
  }
}

static inline int grid_for2(int64_t n, int block, int cap) {
  int64_t g = (n + block - 1) / block;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

}  // namespace dirb200

using namespace dirb200;

extern "C" {

static const int kLossMaxGrid = 1024;

size_t dirb200_loss_workspace_bytes(int64_t n) {
  (void)n;
  return sizeof(double) * kLossMaxGrid + 64;
}

int dirb200_loss_fwd_bwd(int kind, const float* pred, const float* target, const float* weight, int64_t n,
                         float beta, float gamma, int activate, float grad_scale, float* loss_out,
                         float* grad_out, void* workspace, size_t workspace_bytes, void* stream) {
  DIRB_CHECK_ARG(kind >= DIRB200_LOSS_MSE && kind <= DIRB200_LOSS_HUBER, "loss: unknown kind %d", kind);
  DIRB_CHECK_ARG(activate == DIRB200_ACT_SIGMOID || activate == DIRB200_ACT_TANH, "loss: unknown activate %d",
                 activate);
  DIRB_CHECK_ARG(n > 0 && pred && target && loss_out && workspace, "loss: bad arguments");
  if (workspace_bytes < dirb200_loss_workspace_bytes(n)) {
    set_error("loss: workspace too small");
    return DIRB200_ERR_WORKSPACE;
  }
  LossParams p{kind, activate, beta, gamma, grad_scale};
  double* partials = reinterpret_cast<double*>(workspace);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(partials + kLossMaxGrid);
  const int grid = grid_for2(n, 256, kLossMaxGrid);
  if (grid > 1) DIRB_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), as_stream(stream)));
  loss_fwd_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(p, pred, target, weight, n, loss_out, grad_out, partials,
                                                           ticket);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_lds_histogram(const float* labels, int64_t n, int max_target, int64_t* hist, void* stream) {
  DIRB_CHECK_ARG(n >= 0 && max_target > 0 && max_target <= 8192 && hist, "lds_histogram: bad arguments");
  if (n == 0) return DIRB200_OK;
  DIRB_CHECK_ARG(labels, "lds_histogram: null labels");
  lds_hist_kernel<<<grid_for2(n, 256, 2 * num_sms()), 256, sizeof(unsigned int) * max_target, as_stream(stream)>>>(
      labels, n, max_target, reinterpret_cast<unsigned long long*>(hist));
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_lds_table_lookup(const float* values, int64_t n, float mult, int max_bin, const float* table,
                             float* weights_out, void* stream) {
  DIRB_CHECK_ARG(n >= 0 && max_bin >= 0 && table && (n == 0 || (values && weights_out)), "lds_table_lookup: bad arguments");
  if (n == 0) return DIRB200_OK;
  lds_table_lookup_kernel<<<grid_for2(n, 256, 8 * num_sms()), 256, 0, as_stream(stream)>>>(values, n, mult, max_bin,
                                                                                           table, weights_out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_lds_weights_sharded(const float* labels, int64_t n, int64_t n_total, int max_target, int reweight,
                                const double* window_host, int ks, const int64_t* hist, double* scratch,
                                float* weights_out, void* stream) {
  DIRB_CHECK_ARG(reweight == DIRB200_REWEIGHT_SQRT_INV || reweight == DIRB200_REWEIGHT_INVERSE,
                 "lds_weights: reweight must be sqrt_inv or inverse");
  DIRB_CHECK_ARG(n > 0 && n_total >= n && max_target > 0 && max_target <= 8192 && labels && hist && scratch && weights_out,
                 "lds_weights: bad arguments");
  DIRB_CHECK_ARG(ks == 0 || (window_host && ks > 0 && (ks & 1) && ks <= 33), "lds_weights: ks must be 0 or odd <= 33");
  LdsWindow w;
  for (int i = 0; i < 33; ++i) w.w[i] = (i < ks) ? window_host[i] : 0.0;
  for (int i = 0; i < ks / 2; ++i)
    DIRB_CHECK_ARG(window_host[i] == window_host[ks - 1 - i], "lds_weights: window must be symmetric");
  cudaStream_t st = as_stream(stream);
  // the per-bin table and the len / sum(w) normaliser come from the histogram of the WHOLE column (n_total labels)
  lds_bins_kernel<<<1, 128, 0, st>>>(reinterpret_cast<const long long*>(hist), max_target, reweight, w, ks, n_total,
                                     scratch);
  DIRB_LAUNCHED();
  lds_gather_kernel<<<grid_for2(n, 256, 4 * num_sms()), 256, 0, st>>>(labels, n, max_target, scratch, weights_out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int dirb200_lds_weights(const float* labels, int64_t n, int max_target, int reweight, const double* window_host,
                        int ks, const int64_t* hist, double* scratch, float* weights_out, void* stream) {
  return dirb200_lds_weights_sharded(labels, n, n, max_target, reweight, window_host, ks, hist, scratch, weights_out,
                                     stream);
}

}  // extern "C"
