// Bilinear up-sampling arithmetic shared by the standalone up-sampling kernel (dense_ops.cu) and the convolution
// whose A operand is formed from an up-sampled input (conv_igemm.cu): both call these helpers, so the values the
// convolution sees are those dirb200_upsample_bilinear_fwd stores, to the bit.
//
// F.upsample(x, size, mode='bilinear') with align_corners = False (nyud2-dir/models/modules.py:24), as ATen forms it.
// The fma contraction is written out: it is the one nvcc chose for the plain-C++ form of these lines (sm_90a, -O3),
// so no compiler setting can move the rounding of either kernel.
#pragma once
#include <cuda_bf16.h>

namespace dirb200 {

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

}  // namespace dirb200
