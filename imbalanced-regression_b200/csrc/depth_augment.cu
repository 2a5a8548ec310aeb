// Input pipeline of NYUD2-DIR on the device: the per-sample chain of nyud2-dir/loaddata.py:108-125 (with
// nyud2-dir/nyu_transform.py) after Scale(240) --
//     RandomHorizontalFlip -> RandomRotate(5) -> CenterCrop([304, 228], [152, 114]) -> ToTensor -> Lighting(0.1)
//     -> ColorJitter(0.4, 0.4, 0.4) -> Normalize, and the per-pixel loss weight of loaddata.py:58-67
// -- for a whole batch, from uint8 HWC images and uint8 depths (what the host decode + Scale produce) to the fp32
// tensors the network takes.  The random draws are made by the caller with the reference's own generators and passed
// in (flip flags, the rotation as scipy's affine, Lighting's RGB offsets, the jitter order and weights).
//
// Rotation: scipy.ndimage.rotate(a, angle, reshape=False, order=2), mode 'constant', cval 0, on each uint8 plane.
//   * prefilter: the order-2 B-spline filter (one pole) in fp64 along axis 0 (every column), then axis 1 (every row)
//     of each full plane, with scipy's mirror initialisation, its gain and its pole constant, operation for operation;
//   * sampling: only the crop window is evaluated.  Input coordinate = offset + o_y m_0 + o_x m_1 (scipy's order),
//     outside [0, len - 1] on either axis -> cval; the 3 x 3 taps mirror at the edges; sum ((c w_y) w_x) in tap
//     order; uint8 = clip(t + 0.5) truncated.  Every fp64 operation is an explicit _rn intrinsic, so the bytes equal
//     scipy's for the same affine (the host computes the affine with numpy, so cos / sin never run here).
// Depth: Pillow's 8-bit BICUBIC resize (Image.resize default for mode 'L'), horizontal pass then vertical pass, with
//   Pillow's fixed-point coefficients (22 fraction bits) computed here in fp64 the way Pillow computes them, clip8
//   rounding; then ToTensor * 10 and the bucket-weight lookup.  The test chain's 16-bit depth gives int16 / 1000.
// Image: two passes so nothing in fp32 is stored between them.  Pass 1 reduces each image's grayscale sum after the
//   steps that precede Contrast, in fp64 in a fixed order (no atomics); pass 2 recomputes from the uint8 crop and
//   applies Lighting, the jitter in the drawn order with that image's mean, and Normalize, with __fmaf_rn exactly
//   where torch's CPU lerp / add(alpha=) fuse and __fmul_rn / __fadd_rn / __fdiv_rn where it rounds separately.
#include "common.cuh"

namespace dirb200 {

namespace {

// scipy's order-2 pole: the decimal literal -0.171572875253809902396622551580603843 (one ulp from sqrt(8.0) - 3.0)
__device__ __forceinline__ double spline_pole() { return __longlong_as_double(0xbfc5f619980c4337ll); }

constexpr int kGrayBlocks = 16;      // partial sums per image of the grayscale reduction (fixed: no SM dependence)
constexpr int kThreads = 256;

// One line of scipy's apply_filter (ni_splines.c) for one pole with mirror boundaries, in place, stride `st`.
// zn1 = pow(z, n - 1), computed on the host by the C library's pow as scipy does.
__device__ void spline_filter_line(double* c, int n, int64_t st, double zn1) {
  if (n < 2) return;
  const double z = spline_pole();
  const double gain = __dmul_rn(__dsub_rn(1.0, __ddiv_rn(1.0, z)), __dsub_rn(1.0, z));
  for (int i = 0; i < n; ++i) c[i * st] = __dmul_rn(c[i * st], gain);
  // causal initialisation (mirror)
  double c0 = __dadd_rn(__dmul_rn(c[(n - 1) * st], zn1), c[0]);
  double zi = z;
  for (int i = 1; i < n - 1; ++i) {
    const double t = __dmul_rn(__dadd_rn(__dmul_rn(c[(n - 1 - i) * st], zn1), c[i * st]), zi);
    zi = __dmul_rn(zi, z);
    c0 = __dadd_rn(c0, t);
  }
  double prev = __ddiv_rn(c0, __dsub_rn(1.0, __dmul_rn(zn1, zn1)));
  c[0] = prev;
  for (int i = 1; i < n; ++i) {
    prev = __dadd_rn(__dmul_rn(prev, z), c[i * st]);
    c[i * st] = prev;
  }
  // anti-causal initialisation (mirror) and filter
  double last = __ddiv_rn(__dmul_rn(__dadd_rn(__dmul_rn(c[(n - 2) * st], z), prev), z), __dsub_rn(__dmul_rn(z, z), 1.0));
  c[(n - 1) * st] = last;
  for (int i = n - 2; i >= 0; --i) {
    last = __dmul_rn(__dsub_rn(last, c[i * st]), z);
    c[i * st] = last;
  }
}

// axis 0: one thread per (sample, plane, column); loads the (flipped) uint8 source into the fp64 plane first
__global__ void __launch_bounds__(kThreads)
prefilter_cols_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ dep, const uint8_t* __restrict__ flip,
                      int n, int h, int w, double zn1_h, double* __restrict__ coef) {
  const int64_t lines = static_cast<int64_t>(n) * 4 * w;
  for (int64_t l = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; l < lines;
       l += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(l % w);
    const int p = static_cast<int>((l / w) % 4);
    const int b = static_cast<int>(l / (4 * static_cast<int64_t>(w)));
    const int xs = (flip != nullptr && flip[b]) ? w - 1 - x : x;       // FLIP_LEFT_RIGHT before the rotation
    double* c = coef + (static_cast<int64_t>(b) * 4 + p) * h * w + x;
    for (int y = 0; y < h; ++y) {
      const int64_t pix = (static_cast<int64_t>(b) * h + y) * w + xs;
      c[static_cast<int64_t>(y) * w] = static_cast<double>(p < 3 ? img[pix * 3 + p] : dep[pix]);
    }
    spline_filter_line(c, h, w, zn1_h);
  }
}

// axis 1: one thread per (sample, plane, row)
__global__ void __launch_bounds__(kThreads)
prefilter_rows_kernel(int n, int h, int w, double zn1_w, double* __restrict__ coef) {
  const int64_t lines = static_cast<int64_t>(n) * 4 * h;
  for (int64_t l = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; l < lines;
       l += static_cast<int64_t>(gridDim.x) * blockDim.x)
    spline_filter_line(coef + l * w, w, 1, zn1_w);
}

__device__ __forceinline__ int mirror_index(int i, int len) {
  if (len <= 1) return 0;
  const int s2 = 2 * len - 2;
  if (i < 0) {
    i = s2 * (-i / s2) + i;
    i = i <= 1 - len ? i + s2 : -i;
  } else if (i >= len) {
    i -= s2 * (i / s2);
    if (i >= len) i = s2 - i;
  }
  return i;
}

// scipy's get_spline_interpolation_weights, order 2
__device__ __forceinline__ void spline2_weights(double x, double wt[3]) {
  x = __dsub_rn(x, floor(__dadd_rn(x, 0.5)));
  wt[1] = __dsub_rn(0.75, __dmul_rn(x, x));
  const double y = __dsub_rn(0.5, x);
  wt[0] = __dmul_rn(__dmul_rn(0.5, y), y);
  wt[2] = __dsub_rn(__dsub_rn(1.0, wt[0]), wt[1]);
}

// The uint8 crop [n][ch][cw][4] (R, G, B, depth) of the flipped, rotated planes.  coef == NULL: no rotation (a copy).
__global__ void __launch_bounds__(kThreads)
rotate_crop_kernel(const double* __restrict__ coef, const double* __restrict__ affine, const uint8_t* __restrict__ img,
                   const uint8_t* __restrict__ dep, const uint8_t* __restrict__ flip, int n, int h, int w, int y1,
                   int x1, int ch, int cw, uchar4* __restrict__ crop, uchar4* __restrict__ debug_crop) {
  const int64_t total = static_cast<int64_t>(n) * ch * cw;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % cw);
    const int oy = static_cast<int>((i / cw) % ch);
    const int b = static_cast<int>(i / (static_cast<int64_t>(ch) * cw));
    const int ry = oy + y1, rx = ox + x1;                         // pixel of the rotated full-size plane
    uchar4 v = make_uchar4(0, 0, 0, 0);
    if (coef == nullptr) {
      const int xs = (flip != nullptr && flip[b]) ? w - 1 - rx : rx;
      const int64_t pix = (static_cast<int64_t>(b) * h + ry) * w + xs;
      v = make_uchar4(img[pix * 3], img[pix * 3 + 1], img[pix * 3 + 2], dep != nullptr ? dep[pix] : 0);
    } else {
      const double* m = affine + 6 * static_cast<int64_t>(b);
      const double cy = __dadd_rn(__dadd_rn(m[4], __dmul_rn(static_cast<double>(ry), m[0])), __dmul_rn(static_cast<double>(rx), m[1]));
      const double cx = __dadd_rn(__dadd_rn(m[5], __dmul_rn(static_cast<double>(ry), m[2])), __dmul_rn(static_cast<double>(rx), m[3]));
      if (cy >= 0.0 && cy <= static_cast<double>(h - 1) && cx >= 0.0 && cx <= static_cast<double>(w - 1)) {
        double wy[3], wx[3];
        spline2_weights(cy, wy);
        spline2_weights(cx, wx);
        const int sy = static_cast<int>(floor(__dadd_rn(cy, 0.5))) - 1;
        const int sx = static_cast<int>(floor(__dadd_rn(cx, 0.5))) - 1;
        int iy[3], ix[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          iy[k] = mirror_index(sy + k, h);
          ix[k] = mirror_index(sx + k, w);
        }
        uint8_t out[4];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const double* c = coef + (static_cast<int64_t>(b) * 4 + p) * h * w;
          double t = 0.0;
#pragma unroll
          for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int e = 0; e < 3; ++e)
              t = __dadd_rn(t, __dmul_rn(__dmul_rn(c[static_cast<int64_t>(iy[a]) * w + ix[e]], wy[a]), wx[e]));
          double r = __dadd_rn(t, 0.5);
          r = r < 0.0 ? 0.0 : (r > 255.0 ? 255.0 : r);
          out[p] = static_cast<uint8_t>(r);
        }
        v = make_uchar4(out[0], out[1], out[2], out[3]);
      }
    }
    crop[i] = v;
    if (debug_crop != nullptr) debug_crop[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------- photometric chain
struct Photo {
  const float* rgb;         // [n][3] Lighting offsets or NULL
  const int* order;         // [n][3] jitter order (0 brightness, 1 contrast, 2 saturation) or NULL
  const float* alpha;       // [n][3] weight of the k-th applied jitter transform
  float mean[3], stdv[3];   // Normalize
};

__device__ __forceinline__ float gray_of(float r, float g, float b) {
  // Grayscale: gs[0].mul_(0.299).add_(gs[1], alpha=0.587).add_(gs[2], alpha=0.114)
  return __fmaf_rn(0.114f, b, __fmaf_rn(0.587f, g, __fmul_rn(r, 0.299f)));
}

// ToTensor, Lighting and the jitter steps in the drawn order; stop_at_contrast: return before Contrast would run
__device__ __forceinline__ bool photo_chain(const Photo& P, int b, uchar4 u, float x[3], bool stop_at_contrast, float m) {
  x[0] = __fdiv_rn(static_cast<float>(u.x), 255.f);
  x[1] = __fdiv_rn(static_cast<float>(u.y), 255.f);
  x[2] = __fdiv_rn(static_cast<float>(u.z), 255.f);
  if (P.rgb != nullptr) {
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = __fadd_rn(x[c], P.rgb[3 * b + c]);
  }
  if (P.order == nullptr) return false;
  for (int k = 0; k < 3; ++k) {
    const int t = P.order[3 * b + k];
    const float a = P.alpha[3 * b + k];
    if (t == 0) {                        // Brightness: lerp toward 0
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __fmaf_rn(a, __fsub_rn(0.f, x[c]), x[c]);
    } else if (t == 1) {                 // Contrast: lerp toward the image's grayscale mean
      if (stop_at_contrast) return true;
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __fmaf_rn(a, __fsub_rn(m, x[c]), x[c]);
    } else {                             // Saturation: lerp toward the pixel's grayscale
      const float gs = gray_of(x[0], x[1], x[2]);
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __fmaf_rn(a, __fsub_rn(gs, x[c]), x[c]);
    }
  }
  return false;
}

// pass 1: per image, kGrayBlocks partial fp64 sums of the grayscale after the steps preceding Contrast
__global__ void __launch_bounds__(kThreads)
gray_sum_kernel(const uchar4* __restrict__ crop, Photo P, int pixels, double* __restrict__ partial) {
  const int b = blockIdx.y;
  const int chunk = (pixels + kGrayBlocks - 1) / kGrayBlocks;
  const int lo = blockIdx.x * chunk, hi = min(pixels, lo + chunk);
  double s = 0.0;
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    float x[3];
    photo_chain(P, b, crop[static_cast<int64_t>(b) * pixels + i], x, true, 0.f);
    s = __dadd_rn(s, static_cast<double>(gray_of(x[0], x[1], x[2])));
  }
  s = warp_sum(s);
  __shared__ double ws[kThreads / 32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < kThreads / 32; ++k) t = __dadd_rn(t, ws[k]);
    partial[static_cast<int64_t>(b) * kGrayBlocks + blockIdx.x] = t;
  }
}

// pass 2: the whole chain per pixel -> fp32 NCHW
__global__ void __launch_bounds__(kThreads)
photometric_kernel(const uchar4* __restrict__ crop, Photo P, const double* __restrict__ partial, int n, int pixels,
                   float* __restrict__ out, float* __restrict__ debug_mean) {
  const int64_t total = static_cast<int64_t>(n) * pixels;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / pixels);
    const int p = static_cast<int>(i % pixels);
    float m = 0.f;
    if (P.order != nullptr) {
      double s = 0.0;
      for (int k = 0; k < kGrayBlocks; ++k) s = __dadd_rn(s, partial[static_cast<int64_t>(b) * kGrayBlocks + k]);
      m = static_cast<float>(__ddiv_rn(s, static_cast<double>(pixels)));
      if (p == 0 && debug_mean != nullptr) debug_mean[b] = m;
    }
    float x[3];
    photo_chain(P, b, crop[i], x, false, m);
    float* o = out + static_cast<int64_t>(b) * 3 * pixels + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[static_cast<int64_t>(c) * pixels] = __fdiv_rn(__fsub_rn(x[c], P.mean[c]), P.stdv[c]);
  }
}

// ---------------------------------------------------------------------------------------------- depth
__device__ __forceinline__ double bicubic_filter(double x) {      // Pillow's, a = -0.5
  if (x < 0.0) x = -x;
  if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
  if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
  return 0.0;
}

struct ResampleAxis {
  double center, ss;
  int xmin, xmax;            // first source index, tap count
};

// Pillow's precompute_coeffs for one output index (box [0, in_size), bicubic support 2)
__device__ __forceinline__ ResampleAxis resample_axis(int in_size, int out_size, int xx) {
  const double scale = __ddiv_rn(static_cast<double>(in_size), static_cast<double>(out_size));
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(2.0, filterscale);
  ResampleAxis a;
  a.center = __dmul_rn(__dadd_rn(static_cast<double>(xx), 0.5), scale);
  a.ss = __ddiv_rn(1.0, filterscale);
  a.xmin = static_cast<int>(__dadd_rn(__dsub_rn(a.center, support), 0.5));
  if (a.xmin < 0) a.xmin = 0;
  int xmax = static_cast<int>(__dadd_rn(__dadd_rn(a.center, support), 0.5));
  if (xmax > in_size) xmax = in_size;
  a.xmax = xmax - a.xmin;
  return a;
}

__device__ __forceinline__ double resample_weight(const ResampleAxis& a, int x) {
  return bicubic_filter(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + a.xmin), a.center), 0.5), a.ss));
}

__device__ __forceinline__ double resample_total(const ResampleAxis& a) {
  double ww = 0.0;
  for (int x = 0; x < a.xmax; ++x) ww = __dadd_rn(ww, resample_weight(a, x));
  return ww;
}

// normalize_coeffs_8bpc: fixed point with 22 fraction bits
__device__ __forceinline__ int resample_coeff(const ResampleAxis& a, double ww, int x) {
  double k = resample_weight(a, x);
  if (ww != 0.0) k = __ddiv_rn(k, ww);
  return k < 0.0 ? static_cast<int>(__dsub_rn(__dmul_rn(k, 4194304.0), 0.5))
                 : static_cast<int>(__dadd_rn(__dmul_rn(k, 4194304.0), 0.5));
}

__device__ __forceinline__ uint8_t clip8(int in) {
  if (in >= (1 << 30)) return 255;
  if (in <= 0) return 0;
  return static_cast<uint8_t>(in >> 22);
}

// depth [n][1][dh][dw] and weight, from the crop's depth byte (u8 path) or the u16 source (test chain: no resize)
__global__ void __launch_bounds__(kThreads)
depth_kernel(const uchar4* __restrict__ crop, const uint16_t* __restrict__ dep16, int n, int h, int w, int y1, int x1,
             int ch, int cw, int dh, int dw, const float* __restrict__ table, int nb, float* __restrict__ depth,
             float* __restrict__ weight) {
  const int64_t total = static_cast<int64_t>(n) * dh * dw;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % dw);
    const int oy = static_cast<int>((i / dw) % dh);
    const int b = static_cast<int>(i / (static_cast<int64_t>(dh) * dw));
    float d;
    if (dep16 != nullptr) {
      // ToTensor(is_test=True): np.array(pic, np.int16) / 1000
      const uint16_t u = dep16[(static_cast<int64_t>(b) * h + oy + y1) * w + ox + x1];
      d = __fdiv_rn(static_cast<float>(static_cast<int16_t>(u)), 1000.f);
    } else {
      const uchar4* c = crop + static_cast<int64_t>(b) * ch * cw;
      int u;
      if (dh == ch && dw == cw) {
        u = c[static_cast<int64_t>(oy) * cw + ox].w;              // Image.resize to the same size: a copy
      } else {
        const ResampleAxis ay = resample_axis(ch, dh, oy), ax = resample_axis(cw, dw, ox);
        const double wwy = resample_total(ay), wwx = resample_total(ax);
        int acc = 1 << 21;
        for (int ty = 0; ty < ay.xmax; ++ty) {
          const uchar4* row = c + static_cast<int64_t>(ay.xmin + ty) * cw + ax.xmin;
          int hs = 1 << 21;                                        // horizontal pass of this source row
          for (int tx = 0; tx < ax.xmax; ++tx) hs += static_cast<int>(row[tx].w) * resample_coeff(ax, wwx, tx);
          acc += static_cast<int>(clip8(hs)) * resample_coeff(ay, wwy, ty);
        }
        u = clip8(acc);
      }
      d = __fmul_rn(__fdiv_rn(static_cast<float>(u), 255.f), 10.f);   // ToTensor * 10
    }
    depth[i] = d;
    if (weight != nullptr) {
      float wt = 1.f;
      if (table != nullptr) {
        int k = static_cast<int>(__fmul_rn(d, 10.f));             // min(int(d * float32(10)), 99)
        k = k > 99 ? 99 : k;
        wt = table[k];
      }
      weight[i] = wt;
    }
  }
}

inline int grid_for(int64_t items) {
  int64_t g = (items + kThreads - 1) / kThreads;
  const int64_t cap = 32 * static_cast<int64_t>(num_sms());
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

inline size_t align8(size_t b) { return (b + 7) & ~static_cast<size_t>(7); }

struct Layout {
  size_t coef, crop, partial, total;
};

inline Layout layout(int n, int h, int w, int ch, int cw) {
  Layout L;
  L.coef = 0;
  L.crop = align8(static_cast<size_t>(n) * 4 * h * w * sizeof(double));
  L.partial = L.crop + align8(static_cast<size_t>(n) * ch * cw * 4);
  L.total = L.partial + static_cast<size_t>(n) * kGrayBlocks * sizeof(double);
  return L;
}

}  // namespace

}  // namespace dirb200

using namespace dirb200;

extern "C" {

size_t dirb200_depth_augment_workspace_bytes(int n, int h, int w, int crop_h, int crop_w) {
  if (n <= 0 || h <= 0 || w <= 0 || crop_h <= 0 || crop_w <= 0) return 0;
  return layout(n, h, w, crop_h, crop_w).total;
}

int dirb200_depth_augment_batch(const uint8_t* images, const void* depths, int depth_u16, int n, int h, int w,
                                int crop_h, int crop_w, int depth_h, int depth_w, const uint8_t* flip,
                                const double* affine, const float* rgb_offset, const int* jitter_order,
                                const float* jitter_alpha, const float* mean_std, const float* bucket_weights,
                                int n_buckets, float* image_out, float* depth_out, float* weight_out,
                                uint8_t* debug_crop, float* debug_mean, void* workspace, size_t workspace_bytes,
                                void* stream) {
  DIRB_CHECK_ARG(images && depths && image_out && depth_out && mean_std && workspace,
                 "depth_augment_batch: NULL image / depth / output / mean_std / workspace");
  DIRB_CHECK_ARG(n > 0 && h > 0 && w > 0 && crop_h > 0 && crop_w > 0 && depth_h > 0 && depth_w > 0,
                 "depth_augment_batch: sizes must be positive");
  DIRB_CHECK_ARG(crop_h <= h && crop_w <= w, "depth_augment_batch: crop %dx%d larger than the source %dx%d", crop_h,
                 crop_w, h, w);
  DIRB_CHECK_ARG(depth_h <= crop_h && depth_w <= crop_w, "depth_augment_batch: the depth resize only down-samples");
  DIRB_CHECK_ARG(static_cast<int64_t>(n) * h * w * 4 < (static_cast<int64_t>(1) << 31) &&
                     static_cast<int64_t>(h) * w < (static_cast<int64_t>(1) << 31) / 4,
                 "depth_augment_batch: n * h * w * 4 must be below 2^31");
  DIRB_CHECK_ARG(depth_u16 == 0 || depth_u16 == 1, "depth_augment_batch: depth_u16 must be 0 or 1");
  DIRB_CHECK_ARG(!depth_u16 || (affine == nullptr && flip == nullptr && depth_h == crop_h && depth_w == crop_w),
                 "depth_augment_batch: 16-bit depths are the test chain (no flip, rotation or resize)");
  DIRB_CHECK_ARG((jitter_order == nullptr) == (jitter_alpha == nullptr),
                 "depth_augment_batch: jitter_order and jitter_alpha go together");
  DIRB_CHECK_ARG(bucket_weights == nullptr || n_buckets >= 100,
                 "depth_augment_batch: the bucket table needs at least 100 entries (min(int(10 d), 99))");
  DIRB_CHECK_ARG(bucket_weights == nullptr || weight_out != nullptr, "depth_augment_batch: a table needs weight_out");
  const Layout L = layout(n, h, w, crop_h, crop_w);
  DIRB_CHECK_ARG(workspace_bytes >= L.total, "depth_augment_batch: workspace %zu bytes, needs %zu", workspace_bytes,
                 L.total);
  for (int c = 0; c < 3; ++c)
    DIRB_CHECK_ARG(mean_std[3 + c] != 0.f, "depth_augment_batch: std must be non-zero");

  cudaStream_t st = as_stream(stream);
  char* ws = static_cast<char*>(workspace);
  double* coef = reinterpret_cast<double*>(ws + L.coef);
  uchar4* crop = reinterpret_cast<uchar4*>(ws + L.crop);
  double* partial = reinterpret_cast<double*>(ws + L.partial);
  const uint8_t* dep8 = depth_u16 ? nullptr : static_cast<const uint8_t*>(depths);
  // CenterCrop: x1 = int(round((w - tw) / 2.)), Python's round (half to even) = nearbyint
  const int y1 = static_cast<int>(nearbyint((h - crop_h) / 2.0));
  const int x1 = static_cast<int>(nearbyint((w - crop_w) / 2.0));

  if (affine != nullptr) {
    // scipy's z ** (len - 1) for the causal initialisation, by the same C library pow
    const double z = -0.171572875253809902396622551580603843;
    prefilter_cols_kernel<<<grid_for(static_cast<int64_t>(n) * 4 * w), kThreads, 0, st>>>(images, dep8, flip, n, h, w,
                                                                                          pow(z, h - 1), coef);
    DIRB_LAUNCHED();
    prefilter_rows_kernel<<<grid_for(static_cast<int64_t>(n) * 4 * h), kThreads, 0, st>>>(n, h, w, pow(z, w - 1), coef);
    DIRB_LAUNCHED();
  }
  const int64_t pixels = static_cast<int64_t>(crop_h) * crop_w;
  rotate_crop_kernel<<<grid_for(n * pixels), kThreads, 0, st>>>(affine ? coef : nullptr, affine, images, dep8, flip, n,
                                                                h, w, y1, x1, crop_h, crop_w, crop,
                                                                reinterpret_cast<uchar4*>(debug_crop));
  DIRB_LAUNCHED();
  Photo P;
  P.rgb = rgb_offset;
  P.order = jitter_order;
  P.alpha = jitter_alpha;
  for (int c = 0; c < 3; ++c) {
    P.mean[c] = mean_std[c];
    P.stdv[c] = mean_std[3 + c];
  }
  if (jitter_order != nullptr) {
    gray_sum_kernel<<<dim3(kGrayBlocks, n), kThreads, 0, st>>>(crop, P, static_cast<int>(pixels), partial);
    DIRB_LAUNCHED();
  }
  photometric_kernel<<<grid_for(n * pixels), kThreads, 0, st>>>(crop, P, partial, n, static_cast<int>(pixels),
                                                                 image_out, debug_mean);
  DIRB_LAUNCHED();
  depth_kernel<<<grid_for(static_cast<int64_t>(n) * depth_h * depth_w), kThreads, 0, st>>>(
      crop, depth_u16 ? static_cast<const uint16_t*>(depths) : nullptr, n, h, w, y1, x1, crop_h, crop_w, depth_h,
      depth_w, bucket_weights, n_buckets, depth_out, weight_out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
