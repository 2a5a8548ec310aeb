// Internal (C++) interface of the convolution stage shared by conv_igemm.cu, conv_api.cu and the network runner.
#pragma once
#include "common.cuh"

namespace dirb200 {

struct ConvShape {
  int n, h, w, cin, cout, kh, kw, stride, pad, ho, wo;
};

// Which rows of a per-CTA statistics buffer [rows][2][c] hold the partial sums of a channel: the CTAs (or groups of
// `group` CTAs) are dealt round-robin over the n_tiles column tiles of width bn, so channel ch lives in the rows
// (j + k * n_tiles) * group + r   with j = ch / bn, k = 0 .. while the row index < rows, r = 0 .. group-1.
// A plain column reduction over all rows is {rows, 1, c, 1}.
struct StatLayout {
  int rows, n_tiles, bn, group;
};

constexpr int kMaxTaps = 25;   // up to 5x5 filters (the NYUD2 decoder / refinement convs, nyud2-dir/models/modules.py:11-20,154-160)

// One GEMM launch of a conv: the whole conv, or one output-pixel parity class (py, px) of a stride-2 dgrad.
struct ConvLaunch {
  int cls_py, cls_px;           // parity class (stride-2 dgrad only)
  int hm, wm;                   // pixel grid that indexes the GEMM rows
  long long pixels;             // n * hm * wm
  int m_tiles, num_kblocks;
  int grid;                     // persistent CTAs
  int ntaps;                    // filter taps visited ...
  int taps[kMaxTaps];           // ... their indices r*kw + s
  // im2col-mode TMA (a_form 2): GEMM row (y, x) starts at base pixel (y * i2c_stride + i2c_lo, x * i2c_stride + i2c_lo);
  // the base-pixel box of the tensor map runs from (lower_w, lower_h) to the extent plus (upper_w, upper_h)
  int i2c_stride, i2c_lo, i2c_lower_w, i2c_lower_h, i2c_upper_w, i2c_upper_h;
};

// Everything that decides how a conv runs, computed on the host without a CUDA call or an allocation.  conv_fprop,
// conv_dgrad and conv_wgrad_partials execute exactly this plan; dirb200_conv_plan reports it.
struct ConvPlan {
  int op;                       // 0 fprop, 1 dgrad, 2 wgrad
  bool stem;
  int bn, n_tiles;              // GEMM-N tile width and tile count
  int a_form;                   // A operand: 0 cp.async gather, 1 tiled TMA, 2 im2col TMA
  int splits, kblocks_per_split;     // wgrad split-K (else 1, 0)
  size_t workspace_bytes;       // wgrad: the fp32 split-K partials, splits x K x Cout
  bool fuses_bn_moments;        // dgrad: can accumulate the previous layer's BN-backward moments (DgradBnMoments)
  bool classes;                 // stride-2 dgrad: the launches are parity classes ...
  bool need_zero;               // ... and some class has no tap, so dx is zero-filled first
  int nlaunch;
  ConvLaunch launch[4];
  StatLayout layout;            // fprop / stride-1 dgrad: rows of the epilogue's per-CTA statistics
};
// op: 0 fprop, 1 dgrad, 2 wgrad.  Returns the status the launch would return for this shape.
int plan_conv(const ConvShape& s, bool stem, int op, ConvPlan* plan);

// stat_partial (optional): the epilogue also accumulates, per output channel, the sum and the sum of squares of the
// stored outputs into stat_partial[CTA][2][cout] (rows / columns as *layout describes; everything it names is
// written, nothing else is touched) -- the BatchNorm batch statistics without re-reading y.
int conv_fprop(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* y, const ConvShape& s, bool stem,
               cudaStream_t st, float* stat_partial = nullptr, StatLayout* layout = nullptr);
// Inference form (BatchNorm folded into the conv, agedb-dir/resnet.py:46-66 under model.eval()):
//   out = [relu]( conv(x, w) * scale[cout] + shift[cout]  [+ residual] )     -- one launch, no BN pass
struct ConvEpilogue {
  const float* scale;                 // [cout]  gamma / sqrt(running_var + eps)
  const float* shift;                 // [cout]  beta - running_mean * scale
  const __nv_bfloat16* residual;      // optional [pixels][cout] (identity path or the folded downsample branch)
  bool relu;
};
int conv_fprop_affine(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* out, const ConvShape& s,
                      const ConvEpilogue& epi, cudaStream_t st);
// Optional fusion for a dgrad whose output dx is g = d loss / d relu(bn(y)) of the previous conv -> BN -> ReLU layer: the
// epilogue also accumulates that BN's backward moments (sum dz, sum dz*y with dz = g * [y*scale + shift > 0]) into
// partial[CTA][2][cin] (rows as *layout describes), replacing the bn_bwd_reduce pass.  Only where the plan
// fuses_bn_moments (stride 1, TMA-fed A operand).
struct DgradBnMoments {
  const __nv_bfloat16* y;       // raw output of the previous conv, [pixels][cin] like dx
  const float *scale, *shift;   // its BN's forward coefficients (the ReLU mask is re-derived from them)
  float* partial;
  StatLayout* layout;           // out
};
int conv_dgrad(const __nv_bfloat16* dy, const __nv_bfloat16* wt, __nv_bfloat16* dx, const ConvShape& s,
               cudaStream_t st, const DgradBnMoments* bnm = nullptr);
int conv_wgrad_partials(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* partial, const ConvShape& s, bool stem,
                        int* splits_out, cudaStream_t st);
int wgrad_reduce(const float* workspace, int splits, float* dw, const ConvShape& s, bool stem, bool accumulate,
                 cudaStream_t st);
int conv_wgrad(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* dw, float* workspace, const ConvShape& s,
               bool stem, bool accumulate, cudaStream_t st);
struct WgradReduceDesc {        // one conv layer's split-K reduction job (see wgrad_reduce_all)
  const float* partial;         // [splits][cout][kh*kw*cin] (stem: [splits][cout][256]) from conv_wgrad_partials
  size_t w_off;                 // dW (+)= ... at grads + w_off, fp32 [Cout][Cin][KH][KW]
  int splits, cout, cin, kh, kw, stem;
};
int wgrad_reduce_all(const WgradReduceDesc* descs_dev, int nlayers, float* grads, cudaStream_t st);
struct PrepDesc {               // one conv layer's weight re-layout job (see prep_weights_all)
  size_t w_off;                 // fp32 [Cout][Cin][KH][KW] at params + w_off
  int cout, cin, kh, kw, stem;
  __nv_bfloat16 *wf, *wd;       // outputs (wd may be null)
  FastDiv fd_cin, fd_cout, fd_taps;   // reciprocals of cin, cout, kh*kw (make_prep_desc)
};
inline PrepDesc make_prep_desc(size_t w_off, int cout, int cin, int kh, int kw, int stem, __nv_bfloat16* wf,
                               __nv_bfloat16* wd) {
  PrepDesc d{w_off, cout, cin, kh, kw, stem, wf, wd, {}, {}, {}};
  d.fd_cin = make_fastdiv((uint32_t)cin);
  d.fd_cout = make_fastdiv((uint32_t)cout);
  d.fd_taps = make_fastdiv((uint32_t)(kh * kw));
  return d;
}
int prep_weights_all(const float* params, const PrepDesc* descs_dev, int nlayers, cudaStream_t st);
int prep_weights(const float* w, int cout, int cin, int kh, int kw, bool stem, __nv_bfloat16* wf, __nv_bfloat16* wd,
                 cudaStream_t st);
int input_to_s2d(const float* x, int n, int h, int w, __nv_bfloat16* out, cudaStream_t st);

}  // namespace dirb200
