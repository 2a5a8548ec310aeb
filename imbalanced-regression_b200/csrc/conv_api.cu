// C-ABI entry points of the convolution stage + the small layout kernels around
// the wgmma implicit GEMM (weight re-layout, stem space-to-depth, split-K reduce).
#include "common.cuh"
#include "conv.cuh"

namespace dirb200 {

// ---- weights: fp32 [Cout][Cin][KH][KW] (reference / state_dict layout, resnet.py:46-51) ----
//  fprop operand : bf16 [Cout][KH][KW][Cin]      dgrad operand : bf16 [Cin][KH][KW][Cout]
__global__ void prep_weights_kernel(const float* __restrict__ w, int cout, int cin, int kh, int kw,
                                    __nv_bfloat16* __restrict__ wf, __nv_bfloat16* __restrict__ wd) {
  const int64_t total = (int64_t)cout * cin * kh * kw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    // i indexes the fprop layout (coalesced writes): (co, r, s, c)
    int c = (int)(i % cin);
    int64_t t = i / cin;
    int s = (int)(t % kw); t /= kw;
    int r = (int)(t % kh);
    int co = (int)(t / kh);
    const float v = w[(((int64_t)co * cin + c) * kh + r) * kw + s];
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    wf[i] = b;
    if (wd) wd[(((int64_t)c * kh + r) * kw + s) * cout + co] = b;
  }
}

// The stem's GEMM sees the 7x7/2 conv as a 4x4/1 conv over the space-to-depth input: its operand index
// k = (r', s', ph, pw, c4) in [0, 256) is channel c = c4 of the original tap (r, s) = (2 r' + ph - 1, 2 s' + pw - 1).
// false where k holds no weight: c4 == 3 is padding, and r' = 0 with ph = 0 (likewise s', pw) has no tap.
__host__ __device__ __forceinline__ bool stem_tap(int k, int& c, int& r, int& s) {
  const int rp = k >> 6, sp = (k >> 4) & 3, ph = (k >> 3) & 1, pw = (k >> 2) & 1;
  c = k & 3;
  r = 2 * rp + ph - 1;
  s = 2 * sp + pw - 1;
  return c < 3 && r >= 0 && s >= 0;
}

// stem: fp32 [Cout][3][7][7] -> bf16 [Cout][4 r'][4 s'][16 = (ph, pw, c4)] (no tap -> 0)
__global__ void prep_stem_weights_kernel(const float* __restrict__ w, int cout, __nv_bfloat16* __restrict__ wf) {
  const int total = cout * 256;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int co = i >> 8;
    int c, r, s;
    float v = 0.f;
    if (stem_tap(i & 255, c, r, s)) v = w[((co * 3 + c) * 7 + r) * 7 + s];
    wf[i] = __float2bfloat16_rn(v);
  }
}

// x fp32 NCHW [n,3,h,w] -> bf16 [n, h/2, w/2, 16], channel = (ph*2 + pw)*4 + c (c == 3 is zero padding)
__global__ void input_to_s2d_kernel(const float* __restrict__ x, int n, int h, int w, __nv_bfloat16* __restrict__ out) {
  const int h2 = h / 2, w2 = w / 2;
  const int64_t total = (int64_t)n * h2 * w2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int xw = (int)(i % w2);
    const int yh = (int)((i / w2) % h2);
    const int b = (int)(i / ((int64_t)w2 * h2));
    __align__(16) __nv_bfloat16 v[16];
#pragma unroll
    for (int ph = 0; ph < 2; ++ph)
#pragma unroll
      for (int pw = 0; pw < 2; ++pw) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          v[(ph * 2 + pw) * 4 + c] =
              __float2bfloat16_rn(x[(((int64_t)b * 3 + c) * h + (2 * yh + ph)) * w + (2 * xw + pw)]);
        v[(ph * 2 + pw) * 4 + 3] = __float2bfloat16_rn(0.f);
      }
    uint4* o = reinterpret_cast<uint4*>(out + i * 16);
    o[0] = reinterpret_cast<uint4*>(v)[0];
    o[1] = reinterpret_cast<uint4*>(v)[1];
  }
}

// dW[co][c][r][s] (fp32, reference layout) (+)= sum_split partial[split][co][(r*kw+s)*cin + c]
// (partials arrive transposed from the wgrad epilogue: reads are coalesced along k, writes permute (tap, c) -> (c, tap)
// inside one filter's contiguous run)
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int splits, int cout, int cin, int kh, int kw,
                                    int accumulate, float* __restrict__ dw) {
  const int64_t ktot = (int64_t)kh * kw * cin;
  const int64_t total = ktot * cout;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;     // = co * ktot + k
  if (i >= total) return;
  const int co = (int)(i / ktot);
  const int64_t k = i - (int64_t)co * ktot;
  float acc = 0.f;
  for (int sp = 0; sp < splits; ++sp) acc += partial[(int64_t)sp * total + i];
  const int c = (int)(k % cin);
  const int t = (int)(k / cin);
  float* o = dw + ((int64_t)co * cin + c) * (kh * kw) + t;
  *o = accumulate ? *o + acc : acc;
}

__global__ void wgrad_reduce_stem_kernel(const float* __restrict__ partial, int splits, int cout, int accumulate,
                                         float* __restrict__ dw) {
  const int total = 256 * cout;                   // partial[split][co][k], k = (r', s', ph, pw, c4)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int co = i >> 8;
    int c, r, s;
    if (!stem_tap(i & 255, c, r, s)) continue;
    float acc = 0.f;
    for (int sp = 0; sp < splits; ++sp) acc += partial[(int64_t)sp * total + i];
    float* o = dw + ((co * 3 + c) * 7 + r) * 7 + s;
    *o = accumulate ? *o + acc : acc;
  }
}

// Split-K reduction of SEVERAL layers in one launch (blockIdx.y selects the layer, the CTAs of a row stride over its
// weights): the runner keeps one partial buffer per conv and reduces a whole backward stage at once -- 5 launches per
// step instead of 53 latency-bound ones.  Always accumulates into grads (+=), like the per-layer form the runner used.
__global__ void __launch_bounds__(256)
wgrad_reduce_all_kernel(const WgradReduceDesc* __restrict__ descs, float* __restrict__ grads) {
  const WgradReduceDesc d = descs[blockIdx.y];
  float* dw = grads + d.w_off;
  if (d.stem) {
    const int total = 256 * d.cout;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
      const int co = i >> 8;
      int c, r, s;
      if (!stem_tap(i & 255, c, r, s)) continue;
      float acc = 0.f;
      for (int sp = 0; sp < d.splits; ++sp) acc += d.partial[(int64_t)sp * total + i];
      dw[((co * 3 + c) * 7 + r) * 7 + s] += acc;
    }
    return;
  }
  const int64_t ktot = (int64_t)d.kh * d.kw * d.cin;
  const int64_t total = ktot * d.cout;
  const int taps = d.kh * d.kw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float* p = d.partial + i;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;      // four independent chains: the loads of a thread overlap
    int sp = 0;
    for (; sp + 4 <= d.splits; sp += 4) {
      a0 += p[(int64_t)sp * total];
      a1 += p[(int64_t)(sp + 1) * total];
      a2 += p[(int64_t)(sp + 2) * total];
      a3 += p[(int64_t)(sp + 3) * total];
    }
    for (; sp < d.splits; ++sp) a0 += p[(int64_t)sp * total];
    const int64_t co = i / ktot, k = i - co * ktot;
    const int c = (int)(k % d.cin), t = (int)(k / d.cin);
    dw[(co * d.cin + c) * taps + t] += (a0 + a1) + (a2 + a3);
  }
}

int wgrad_reduce_all(const WgradReduceDesc* descs_dev, int nlayers, float* grads, cudaStream_t st) {
  if (nlayers <= 0) return DIRB200_OK;
  wgrad_reduce_all_kernel<<<dim3(2 * num_sms(), nlayers), 256, 0, st>>>(descs_dev, grads);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

// All conv weights of a network in ONE launch: blockIdx.y selects the layer.
__global__ void prep_weights_all_kernel(const float* __restrict__ params, const PrepDesc* __restrict__ descs) {
  const PrepDesc d = descs[blockIdx.y];
  const float* w = params + d.w_off;
  if (d.stem) {
    const int total = d.cout * 256;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
      const int co = i >> 8;
      int c, r, s;
      float v = 0.f;
      if (stem_tap(i & 255, c, r, s)) v = w[((co * 3 + c) * 7 + r) * 7 + s];
      d.wf[i] = __float2bfloat16_rn(v);
    }
    return;
  }
  // Two coalesced-store passes (one thread per OUTPUT element; the fp32 source is gathered, its 32-byte sectors are
  // shared by neighbouring threads through L1/L2) instead of one pass with 2-byte scattered stores into the transposed
  // copy; index arithmetic by multiply-high reciprocals filled in on the host.
  const uint32_t taps = (uint32_t)(d.kh * d.kw);
  const uint32_t total = (uint32_t)d.cout * (uint32_t)d.cin * taps;
  const uint32_t stride = gridDim.x * blockDim.x;
  // fprop operand [co][tap][c]
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    uint32_t t, c, co, tap;
    d.fd_cin.divmod(i, t, c);
    d.fd_taps.divmod(t, co, tap);
    d.wf[i] = __float2bfloat16_rn(w[((size_t)co * d.cin + c) * taps + tap]);
  }
  if (!d.wd) return;
  // dgrad operand [c][tap][co]
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    uint32_t t, c, co, tap;
    d.fd_cout.divmod(i, t, co);
    d.fd_taps.divmod(t, c, tap);
    d.wd[i] = __float2bfloat16_rn(w[((size_t)co * d.cin + c) * taps + tap]);
  }
}

int prep_weights_all(const float* params, const PrepDesc* descs_dev, int nlayers, cudaStream_t st) {
  prep_weights_all_kernel<<<dim3(96, nlayers), 256, 0, st>>>(params, descs_dev);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

static inline int grid1d(int64_t n, int block = 256) {
  int64_t g = (n + block - 1) / block;
  const int64_t cap = 8 * (int64_t)num_sms();
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

int prep_weights(const float* w, int cout, int cin, int kh, int kw, bool stem, __nv_bfloat16* wf, __nv_bfloat16* wd,
                 cudaStream_t st) {
  if (stem) {
    prep_stem_weights_kernel<<<grid1d((int64_t)cout * 256), 256, 0, st>>>(w, cout, wf);
  } else {
    prep_weights_kernel<<<grid1d((int64_t)cout * cin * kh * kw), 256, 0, st>>>(w, cout, cin, kh, kw, wf, wd);
  }
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int input_to_s2d(const float* x, int n, int h, int w, __nv_bfloat16* out, cudaStream_t st) {
  input_to_s2d_kernel<<<grid1d((int64_t)n * (h / 2) * (w / 2)), 256, 0, st>>>(x, n, h, w, out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int wgrad_reduce(const float* workspace, int splits, float* dw, const ConvShape& s, bool stem, bool accumulate,
                 cudaStream_t st) {
  if (stem)
    wgrad_reduce_stem_kernel<<<grid1d(256 * (int64_t)s.cout), 256, 0, st>>>(workspace, splits, s.cout, accumulate, dw);
  else
  {
    // latency-bound gather/scatter: one thread per weight so that every load is in flight at once
    const int64_t total = (int64_t)s.kh * s.kw * s.cin * s.cout;
    wgrad_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(workspace, splits, s.cout, s.cin, s.kh, s.kw,
                                                                         accumulate, dw);
  }
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

int conv_wgrad(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* workspace, const ConvShape& s,
               bool stem, bool accumulate, cudaStream_t st) {
  int splits = 1;
  if (int rc = conv_wgrad_partials(x, dy, workspace, s, stem, &splits, st)) return rc;
  return wgrad_reduce(workspace, splits, dw, s, stem, accumulate, st);
}

// API shape (original conv hyper-parameters) -> kernel shape.  The stem (cin = 3, 7x7, stride 2, pad 3) runs
// as a 4x4 / stride-1 / pad-2 conv over the 16-channel space-to-depth input.
static int to_shape(int n, int h, int w, int cin, int cout, int kh, int kw, int stride, int pad, int stem,
                    ConvShape* s) {
  if (stem) {
    DIRB_CHECK_ARG(cin == 3 && kh == 7 && kw == 7 && stride == 2 && pad == 3 && h % 2 == 0 && w % 2 == 0,
                   "stem conv must be 3->Cout 7x7 stride 2 pad 3 on even H, W");
    *s = ConvShape{n, h / 2, w / 2, 16, cout, 4, 4, 1, 2, h / 2, w / 2};
  } else {
    DIRB_CHECK_ARG(n > 0 && h > 0 && w > 0 && kh > 0 && kw > 0 && stride > 0 && pad >= 0, "bad conv shape");
    *s = ConvShape{n, h, w, cin, cout, kh, kw, stride, pad, (h + 2 * pad - kh) / stride + 1,
                   (w + 2 * pad - kw) / stride + 1};
  }
  return DIRB200_OK;
}

/* ---- Test aids: the runner's batched weight re-layout and split-K reduction, one launch over caller-given jobs (see
 * include/dirb200.h).  The jobs become the runner's own descriptors (make_prep_desc, WgradReduceDesc) in a device table
 * that lives in stream order around the launch. */
static int conv_job_shape_ok(const char* who, int k, int cout, int cin, int kh, int kw, int stem) {
  DIRB_CHECK_ARG(cout > 0 && cin > 0 && kh > 0 && kw > 0, "%s: job %d has a non-positive size (%d, %d, %d, %d)", who, k,
                 cout, cin, kh, kw);
  DIRB_CHECK_ARG(!stem || (cin == 3 && kh == 7 && kw == 7), "%s: job %d: the stem must be 3x7x7", who, k);
  const int64_t weights = (int64_t)cout * cin * kh * kw;
  DIRB_CHECK_ARG(weights < (int64_t(1) << 31) && (!stem || 256 * (int64_t)cout < (int64_t(1) << 31)),
                 "%s: job %d has 2^31 or more weights", who, k);
  return DIRB200_OK;
}

}  // namespace dirb200

using namespace dirb200;

extern "C" {

int dirb200_conv_prep_weights(const float* w, int cout, int cin, int kh, int kw, int stem, void* w_fprop,
                              void* w_dgrad, void* stream) {
  DIRB_CHECK_ARG(w && w_fprop && cout > 0 && cin > 0, "conv_prep_weights: bad arguments");
  DIRB_CHECK_ARG(!stem || (cin == 3 && kh == 7 && kw == 7), "conv_prep_weights: stem must be 3x7x7");
  return prep_weights(w, cout, cin, kh, kw, stem != 0, (__nv_bfloat16*)w_fprop, (__nv_bfloat16*)w_dgrad,
                      as_stream(stream));
}

int dirb200_input_to_s2d(const float* x_nchw, int n, int h, int w, void* out_bf16, void* stream) {
  DIRB_CHECK_ARG(x_nchw && out_bf16 && n > 0 && h > 0 && w > 0 && h % 2 == 0 && w % 2 == 0,
                 "input_to_s2d: bad arguments");
  return input_to_s2d(x_nchw, n, h, w, (__nv_bfloat16*)out_bf16, as_stream(stream));
}

int dirb200_conv_fprop(const void* x, const void* w_fprop, void* y, int n, int h, int w, int cin, int cout, int kh,
                       int kw, int stride, int pad, int stem, void* stream) {
  DIRB_CHECK_ARG(x && w_fprop && y, "conv_fprop: null pointer");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, stem, &s)) return rc;
  return conv_fprop((const __nv_bfloat16*)x, (const __nv_bfloat16*)w_fprop, (__nv_bfloat16*)y, s, stem != 0,
                    as_stream(stream));
}

int dirb200_conv_dgrad(const void* dy, const void* w_dgrad, void* dx, int n, int h, int w, int cin, int cout, int kh,
                       int kw, int stride, int pad, void* stream) {
  DIRB_CHECK_ARG(dy && w_dgrad && dx, "conv_dgrad: null pointer");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, 0, &s)) return rc;
  return conv_dgrad((const __nv_bfloat16*)dy, (const __nv_bfloat16*)w_dgrad, (__nv_bfloat16*)dx, s,
                    as_stream(stream));
}

size_t dirb200_conv_wgrad_workspace_bytes(int n, int h, int w, int cin, int cout, int kh, int kw, int stride, int pad,
                                          int stem) {
  ConvShape s;
  ConvPlan pl;
  if (to_shape(n, h, w, cin, cout, kh, kw, stride, pad, stem, &s) || plan_conv(s, stem != 0, 2, &pl)) return 0;
  return pl.workspace_bytes;
}

int dirb200_conv_wgrad(const void* x, const void* dy, float* dw, void* workspace, size_t workspace_bytes, int n, int h,
                       int w, int cin, int cout, int kh, int kw, int stride, int pad, int stem, int accumulate,
                       void* stream) {
  DIRB_CHECK_ARG(x && dy && dw && workspace, "conv_wgrad: null pointer");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, stem, &s)) return rc;
  ConvPlan pl;
  if (int rc = plan_conv(s, stem != 0, 2, &pl)) return rc;
  if (workspace_bytes < pl.workspace_bytes) {
    set_error("conv_wgrad: workspace too small (%zu < %zu)", workspace_bytes, pl.workspace_bytes);
    return DIRB200_ERR_WORKSPACE;
  }
  return conv_wgrad((const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, dw, (float*)workspace, s, stem != 0,
                    accumulate != 0, as_stream(stream));
}

/* ---- Test aids: the fused epilogues the network runner uses, one call each (see include/dirb200.h). */
static void layout_to_host(const StatLayout& l, int* layout_host) {
  layout_host[0] = l.rows; layout_host[1] = l.n_tiles; layout_host[2] = l.bn; layout_host[3] = l.group;
}

int dirb200_conv_fprop_bn_stats(const void* x, const void* w_fprop, void* y, int n, int h, int w, int cin, int cout,
                                int kh, int kw, int stride, int pad, int stem, float* partial, int* layout_host,
                                void* stream) {
  DIRB_CHECK_ARG(x && w_fprop && y && partial && layout_host, "conv_fprop_bn_stats: null pointer");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, stem, &s)) return rc;
  StatLayout lay{};
  if (int rc = conv_fprop((const __nv_bfloat16*)x, (const __nv_bfloat16*)w_fprop, (__nv_bfloat16*)y, s, stem != 0,
                          as_stream(stream), partial, &lay))
    return rc;
  layout_to_host(lay, layout_host);
  return DIRB200_OK;
}

int dirb200_conv_fprop_affine(const void* x, const void* w_fprop, void* out, int n, int h, int w, int cin, int cout,
                              int kh, int kw, int stride, int pad, const float* scale, const float* shift,
                              const void* residual, int relu, void* stream) {
  DIRB_CHECK_ARG(x && w_fprop && out, "conv_fprop_affine: null pointer");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, 0, &s)) return rc;
  return conv_fprop_affine((const __nv_bfloat16*)x, (const __nv_bfloat16*)w_fprop, (__nv_bfloat16*)out, s,
                           ConvEpilogue{scale, shift, (const __nv_bfloat16*)residual, relu != 0}, as_stream(stream));
}

int dirb200_conv_dgrad_bn_moments(const void* dy, const void* w_dgrad, void* dx, int n, int h, int w, int cin, int cout,
                                  int kh, int kw, int stride, int pad, const void* y_prev, const float* scale,
                                  const float* shift, float* partial, int* layout_host, void* stream) {
  DIRB_CHECK_ARG(dy && w_dgrad && dx && y_prev && scale && shift && partial && layout_host,
                 "conv_dgrad_bn_moments: null pointer");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, 0, &s)) return rc;
  StatLayout lay{};
  const DgradBnMoments bm{(const __nv_bfloat16*)y_prev, scale, shift, partial, &lay};
  if (int rc = conv_dgrad((const __nv_bfloat16*)dy, (const __nv_bfloat16*)w_dgrad, (__nv_bfloat16*)dx, s,
                          as_stream(stream), &bm))
    return rc;
  layout_to_host(lay, layout_host);
  return DIRB200_OK;
}

/* Host-only (no CUDA call): the plan dirb200_conv_fprop / _dgrad / _wgrad (op 0 / 1 / 2) would execute for this
 * shape, or the status they would refuse it with: plan7[0] tile width BN, [1] 0 (no CTA pairs), [2] A-operand form (0 cp.async gather, 1 tiled TMA, 2 im2col
 * TMA), [3] 0 (no patch-resident form), [4] split-K factor, [5] launches, [6] dgrad can carry the BN-backward moments of
 * the previous layer. */
int dirb200_conv_plan(int n, int h, int w, int cin, int cout, int kh, int kw, int stride, int pad, int stem, int op,
                      int* plan7) {
  DIRB_CHECK_ARG(plan7 && op >= 0 && op <= 2, "conv_plan: bad arguments");
  ConvShape s;
  if (int rc = to_shape(n, h, w, cin, cout, kh, kw, stride, pad, stem, &s)) return rc;
  ConvPlan pl;
  if (int rc = plan_conv(s, stem != 0, op, &pl)) return rc;
  const int v[7] = {pl.bn, 0, pl.a_form, 0, pl.splits, pl.nlaunch, pl.fuses_bn_moments ? 1 : 0};
  for (int i = 0; i < 7; ++i) plan7[i] = v[i];
  return DIRB200_OK;
}

int dirb200_prep_weights_all(const float* params, const dirb200_prep_job* jobs_host, int njobs, void* stream) {
  DIRB_CHECK_ARG(params && jobs_host, "prep_weights_all: null pointer");
  DIRB_CHECK_ARG(njobs >= 1 && njobs <= 65535, "prep_weights_all: njobs must be 1 .. 65535 (got %d)", njobs);
  std::vector<PrepDesc> descs;
  for (int k = 0; k < njobs; ++k) {
    const dirb200_prep_job& j = jobs_host[k];
    DIRB_CHECK_ARG(j.w_fprop, "prep_weights_all: job %d has a null w_fprop", k);
    DIRB_CHECK_ARG(j.w_off >= 0, "prep_weights_all: job %d has a negative w_off", k);
    if (int rc = conv_job_shape_ok("prep_weights_all", k, j.cout, j.cin, j.kh, j.kw, j.stem)) return rc;
    DIRB_CHECK_ARG(!j.stem || !j.w_dgrad, "prep_weights_all: job %d: the stem has no dgrad operand (w_dgrad must be null)",
                   k);
    descs.push_back(make_prep_desc((size_t)j.w_off, j.cout, j.cin, j.kh, j.kw, j.stem ? 1 : 0,
                                   (__nv_bfloat16*)j.w_fprop, (__nv_bfloat16*)j.w_dgrad));
  }
  cudaStream_t st = as_stream(stream);
  return with_device_table(descs, st, [&](const PrepDesc* d) { return prep_weights_all(params, d, njobs, st); });
}

int dirb200_wgrad_reduce_all(const dirb200_wgrad_reduce_job* jobs_host, int njobs, float* grads, void* stream) {
  DIRB_CHECK_ARG(jobs_host && grads, "wgrad_reduce_all: null pointer");
  DIRB_CHECK_ARG(njobs >= 1 && njobs <= 65535, "wgrad_reduce_all: njobs must be 1 .. 65535 (got %d)", njobs);
  std::vector<WgradReduceDesc> descs;
  for (int k = 0; k < njobs; ++k) {
    const dirb200_wgrad_reduce_job& j = jobs_host[k];
    DIRB_CHECK_ARG(j.partial, "wgrad_reduce_all: job %d has a null partial", k);
    DIRB_CHECK_ARG(j.w_off >= 0, "wgrad_reduce_all: job %d has a negative w_off", k);
    DIRB_CHECK_ARG(j.splits >= 1, "wgrad_reduce_all: job %d: splits must be at least 1 (got %d)", k, j.splits);
    if (int rc = conv_job_shape_ok("wgrad_reduce_all", k, j.cout, j.cin, j.kh, j.kw, j.stem)) return rc;
    descs.push_back(WgradReduceDesc{j.partial, (size_t)j.w_off, j.splits, j.cout, j.cin, j.kh, j.kw, j.stem ? 1 : 0});
  }
  cudaStream_t st = as_stream(stream);
  return with_device_table(descs, st, [&](const WgradReduceDesc* d) { return wgrad_reduce_all(d, njobs, grads, st); });
}

}  // extern "C"
