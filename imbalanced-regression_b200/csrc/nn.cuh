// Internal (C++) interface of the HBM-bound ResNet layers (nn_kernels.cu).
#pragma once
#include "common.cuh"
#include "conv.cuh"

namespace dirb200 {

int bn_partial_floats(int max_c);   // size of the per-CTA partial buffer shared by the column reductions
int bn_stats(const __nv_bfloat16* y, int64_t rows, int c, float* partial, int* nblocks, cudaStream_t st);
// partial: [rows][2][c] column sums / sums of squares, rows per channel as `layout` says (conv.cuh)
int bn_finalize(const float* partial, const StatLayout& layout, int64_t rows, int c, const float* gamma, const float* beta,
                float eps, float momentum, float* running_mean, float* running_var, float* mean, float* invstd,
                float* scale, float* shift, cudaStream_t st);
struct BnEvalDesc {            // one BN layer of the network (bn_eval_coeffs_all)
  int c;
  size_t gamma_off, beta_off;  // in the flat parameter buffer (floats)
  size_t rm_off, rv_off;       // in the flat running-statistics buffer (floats)
  float *scale, *shift;        // outputs [c]
};
// eval-mode scale / shift of EVERY BN layer in one launch
int bn_eval_coeffs_all(const BnEvalDesc* descs_dev, int nlayers, int max_c, const float* params, const float* running,
                       float eps, cudaStream_t st);
int bn_eval_coeffs(int c, const float* gamma, const float* beta, float eps, const float* running_mean,
                   const float* running_var, float* scale, float* shift, cudaStream_t st);
// mask_out (optional): [rows][c/8] bytes, bit j of byte (r, cg) = out[r][cg*8+j] > 0
int bn_apply(const __nv_bfloat16* y, const float* scale, const float* shift, const __nv_bfloat16* res,
             const __nv_bfloat16* res_y, const float* res_scale, const float* res_shift, bool relu, int64_t rows, int c,
             __nv_bfloat16* out, uint8_t* mask_out, cudaStream_t st);
// BN backward, ReLU mask from (y, scale, shift) when mask == nullptr, else from the stored bit mask
// g2_h, g2_w > 0: g2 is the COMPACT [n, g2_h/2, g2_w/2, c] gradient of a stride-2 1x1 downsample conv (added at even y, x)
// dz_out (identity blocks): dz = (g1 [+ g2]) * mask is stored and summed as stored; bn_bwd_apply then takes dz as its
// only gradient input (mask == scale == shift == nullptr)
// g3 (with g2 and dz_out only): a third dense gradient, summed in fp32 with g1 + g2 before dz is rounded to bf16
int bn_bwd_reduce(const __nv_bfloat16* g1, const __nv_bfloat16* g2, const __nv_bfloat16* y, const __nv_bfloat16* y2,
                  const float* scale, const float* shift, const uint8_t* mask, int64_t rows, int c, float* partial,
                  int* nblocks, cudaStream_t st, int g2_h = 0, int g2_w = 0, __nv_bfloat16* dz_out = nullptr,
                  const __nv_bfloat16* g3 = nullptr);
int bn_bwd_coeffs(const float* partial, int nblocks, int k, int gslot, int64_t rows, int c, const float* mean,
                  const float* invstd, const float* gamma, float* grad_gamma, float* grad_beta, float* coef,
                  cudaStream_t st);
// the same coefficients from the moments a dgrad epilogue accumulated (conv_dgrad with DgradBnMoments)
int bn_bwd_coeffs_layout(const float* partial, const StatLayout& layout, int64_t rows, int c, const float* mean,
                         const float* invstd, const float* gamma, float* grad_gamma, float* grad_beta, float* coef,
                         cudaStream_t st);
int bn_bwd_apply(const __nv_bfloat16* g1, const __nv_bfloat16* g2, const __nv_bfloat16* y, const float* coef,
                 const __nv_bfloat16* y2, const float* coef2, const float* scale, const float* shift,
                 const uint8_t* mask, int64_t rows, int c, __nv_bfloat16* dy, __nv_bfloat16* dy2,
                 __nv_bfloat16* dz_out, cudaStream_t st, int g2_h = 0, int g2_w = 0);
// stem: relu(bn(y)) + 3x3/2 max pool in one pass (the activation itself is not materialised)
int bn_relu_maxpool_fwd(const __nv_bfloat16* y, const float* scale, const float* shift, int n, int h, int w, int c,
                        __nv_bfloat16* out, uint8_t* idx, cudaStream_t st);
int maxpool_fwd(const __nv_bfloat16* x, int n, int h, int w, int c, __nv_bfloat16* out, uint8_t* idx, cudaStream_t st);
int maxpool_bwd(const __nv_bfloat16* g1, const __nv_bfloat16* g2, const uint8_t* idx, int n, int h, int w, int c,
                __nv_bfloat16* dx, cudaStream_t st);
int avgpool_fwd(const __nv_bfloat16* x, int n, int hw, int c, float* enc, cudaStream_t st);
int avgpool_bwd(const float* genc, int n, int hw, int c, __nv_bfloat16* dx, cudaStream_t st);

}  // namespace dirb200
