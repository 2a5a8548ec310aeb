// Label -> bin rules shared by the FDS kernels (fds.cu) and the STS-B shot metrics (metrics.cu).
#pragma once
#include "common.cuh"

namespace dirb200 {

// Row label -> table row (bucket - bucket_start), -1 = row not touched.
//   rule 0 (age, agedb-dir/fds.py:91-104): int(label - bucket_start); out-of-range labels fold into an edge bin only
//           when the edge value itself occurs among the labels (has_lo / has_hi).
//   rule 1 (depth, nyud2-dir/models/fds.py:51-53): clamp(int(label * 10), bucket_start, bucket_num - 1).
//   rule 2 (STS-B, sts-b-dir/fds.py:51-57): np.histogram edges over [0, 5] with bucket_num bins: the bucket whose
//           half-open edge interval holds the label (label == 5 -> last), clamped below by bucket_start.
__device__ __forceinline__ int bin_of(int rule, float v, float lo, float hi, int nb, bool has_lo, bool has_hi) {
  if (rule == DIRB200_BIN_AGE) {
    if (v < lo) return has_lo ? 0 : -1;
    if (v > hi) return has_hi ? nb - 1 : -1;
    if (!(v >= lo)) return -1;  // NaN
    return (int)(v - lo);       // int(label - bucket_start), fds.py:104
  }
  const int start = (int)lo, last = (int)hi;       // bucket_start, bucket_num - 1
  if (!(v == v)) return -1;
  int b;
  if (rule == DIRB200_BIN_DEPTH10) {
    b = (int)__fmul_rn(v, 10.0f);
  } else {
    const int num = last + 1;
    if (v >= 5.0f) {
      b = last;                                     // label == 5. -> bucket_num - 1 (labels > 5 are out of contract)
    } else {
      // edges e_i = float32(i * (5 / num)) (np.linspace in float64, cast to the float32 label dtype)
      const double step = 5.0 / (double)num;
      b = (int)floor((double)v / step);
      if (b < 0) b = 0;
      if (b > last) b = last;
      while (b < last && (float)((double)(b + 1) * step) <= v) ++b;     // first edge > label is e_{b+1}
      while (b > 0 && (float)((double)b * step) > v) --b;
    }
  }
  b = max(start, min(last, b));
  return b - start;
}

}  // namespace dirb200
