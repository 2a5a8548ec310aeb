// JPEG decode and Pillow's bilinear resize on the device: the host stages of agedb-dir/datasets.py:30, :41 and :49,
// Image.open(f).convert('RGB') then transforms.Resize((S, S)), for a batch of images of mixed sizes, byte for byte as
// Pillow built on libjpeg-turbo computes them.
//
// Host: dirb200_jpeg_parse walks the markers (no CUDA call) and keeps the raw DQT / DHT arrays, the sampling factors
//   and the start of every restart interval.  Anything outside the supported set is left to the host decoder.
// Device, per batch:
//   plan      one CTA: validates each descriptor against its byte range and output slice, checks its Huffman tables,
//             and lays the batch out in the workspace (exclusive scans of blocks and intervals);
//   tables    per image and Huffman table: libjpeg's derived table (maxcode / valoffset) plus a 9-bit lookahead;
//   entropy   one thread per restart interval: stuffed 0xFF00 removed on the fly, DC prediction restarting at each
//             interval, de-zigzagged int16 coefficients (libjpeg's JCOEF).  Anomalies set the image's status;
//   idct      one thread per 8 x 8 block: dequantisation and jidctint.c's JDCT_ISLOW (CONST_BITS 13, PASS1_BITS 2)
//             with its range-limit table, index masked with 0x3FF.  A block whose values leave the range in which
//             libjpeg-turbo's 16-bit SIMD IDCT gives the same result sets the image's status;
//   colour    one thread per output pixel: libjpeg-turbo's fancy h2v1 / h2v2 triangle upsampling over the chroma's
//             downsampled width (edge rows repeated as libjpeg's context rows are), jdcolor.c's YCbCr -> RGB with
//             SCALEBITS 16; grayscale is replicated to three channels as convert('RGB') does.
// Resize: Pillow's ImagingResample, 8 bits per channel: per output index a window and weights in double, normalised,
// turned into 22-bit fixed point with Pillow's rounding (coefficient kernel), then the horizontal pass into an 8-bit
// value per source row the vertical pass reads, then the vertical pass (one thread per output pixel).
#include "common.cuh"
#include <cub/block/block_scan.cuh>
#include <string.h>

namespace dirb200 {

namespace {

typedef dirb200_jpeg_desc Desc;

// jpeg_natural_order: natural index of the k-th coefficient in zigzag order
constexpr uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_natural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                      12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                      35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                      58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

__host__ __device__ __forceinline__ int kNaturalAt(int k) {
#ifdef __CUDA_ARCH__
  return c_natural[k];
#else
  return kNatural[k];
#endif
}

constexpr int64_t kMaxPixels = int64_t(1) << 26;

// status bits
constexpr int kBadDesc = 1;        // descriptor outside the supported set, its byte range or its output slice
constexpr int kBadCode = 2;        // a code that is not in the Huffman table
constexpr int kOverrun = 4;        // entropy-coded data ran out (the decode consumed bits past a marker / range end)
constexpr int kTooMany = 8;        // a coefficient past position 63 of a block
constexpr int kWorkspace = 16;     // the workspace does not hold the batch
constexpr int kIdctRange = 32;     // a block outside the range in which libjpeg-turbo's SIMD and C IDCTs agree

// ---------------------------------------------------------------------------------------------- shared descriptor rules
__host__ __device__ inline int comp_blocks_w(const Desc& d, int c) { return d.ncomp == 1 ? d.mcus_x : d.mcus_x * d.comp_h[c]; }
__host__ __device__ inline int comp_blocks_h(const Desc& d, int c) { return d.ncomp == 1 ? d.mcus_y : d.mcus_y * d.comp_v[c]; }

__host__ __device__ inline int64_t image_blocks(const Desc& d) {
  int64_t b = 0;
  for (int c = 0; c < d.ncomp; ++c) b += static_cast<int64_t>(comp_blocks_w(d, c)) * comp_blocks_h(d, c);
  return b;
}

// jpeg_make_d_derived_tbl's checks: at most 256 symbols, no code of all ones, DC symbols 0..15
__host__ __device__ inline bool huff_table_ok(const uint8_t* bits, const uint8_t* vals, bool dc) {
  int p = 0;
  uint32_t code = 0;
  for (int l = 1; l <= 16; ++l) {
    p += bits[l - 1];
    if (p > 256) return false;
    code += bits[l - 1];
    if (code >= (1u << l)) return false;   // one past this length's last code must still fit in l bits
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < p; ++i)
      if (vals[i] > 15) return false;
  return true;
}

// the supported set, restated on the device from whatever the caller passed
__host__ __device__ inline bool desc_ok(const Desc& d) {
  if (d.width < 1 || d.height < 1 || d.width > 65535 || d.height > 65535) return false;
  if (static_cast<int64_t>(d.width) * d.height > kMaxPixels) return false;
  if (d.ncomp == 1) {
    if (d.comp_h[0] != 1 || d.comp_v[0] != 1 || d.hmax != 1 || d.vmax != 1) return false;
  } else if (d.ncomp == 3) {
    const int h = d.comp_h[0], v = d.comp_v[0];
    if (!((h == 1 && v == 1) || (h == 2 && v == 1) || (h == 2 && v == 2))) return false;
    if (d.hmax != h || d.vmax != v) return false;
    for (int c = 1; c < 3; ++c)
      if (d.comp_h[c] != 1 || d.comp_v[c] != 1) return false;
  } else {
    return false;
  }
  const int mx = (d.width + 8 * d.hmax - 1) / (8 * d.hmax), my = (d.height + 8 * d.vmax - 1) / (8 * d.vmax);
  if (d.mcus_x != mx || d.mcus_y != my) return false;
  const int64_t mcus = static_cast<int64_t>(mx) * my;
  if (d.restart_interval < 0 || d.restart_interval > 65535) return false;
  const int64_t iv = d.restart_interval ? (mcus + d.restart_interval - 1) / d.restart_interval : 1;
  if (d.n_intervals != iv) return false;
  if (d.scan_begin < 0 || d.scan_end < d.scan_begin) return false;
  for (int c = 0; c < d.ncomp; ++c) {
    if (d.comp_tq[c] < 0 || d.comp_tq[c] > 3 || d.comp_td[c] < 0 || d.comp_td[c] > 3 || d.comp_ta[c] < 0 ||
        d.comp_ta[c] > 3)
      return false;
    if (!huff_table_ok(d.huff_bits[0][d.comp_td[c]], d.huff_vals[0][d.comp_td[c]], true)) return false;
    if (!huff_table_ok(d.huff_bits[1][d.comp_ta[c]], d.huff_vals[1][d.comp_ta[c]], false)) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------- workspace layout
struct ImgPlan {
  int64_t coef;       // element offset of the image's int16 coefficients (component 0 first)
  int64_t plane;      // byte offset of its component planes
  int64_t iv0;        // its first entry in the batch's interval table
  int32_t ok;         // descriptor usable (status had no kBadDesc / kWorkspace)
  int32_t pad;
};

// libjpeg's derived table plus a 9-bit lookahead: look[i] = (length << 8) | symbol for the code that prefixes i
struct HuffTab {
  uint16_t look[512];
  int32_t maxcode[18];
  int32_t valoff[18];
  uint8_t vals[256];
};

constexpr int kLookBits = 9;

inline __host__ __device__ size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

struct DecodeLayout {
  size_t plans, tabs, coef, fixed;
};
inline __host__ __device__ DecodeLayout decode_layout(int n) {
  DecodeLayout L;
  L.plans = 0;
  L.tabs = align256(static_cast<size_t>(n) * sizeof(ImgPlan));
  L.coef = L.tabs + align256(static_cast<size_t>(n) * 8 * sizeof(HuffTab));
  L.fixed = L.coef;
  return L;
}
// after the fixed part: coefficients (128 bytes per block) then planes (64 bytes per block)
inline __host__ __device__ size_t decode_ws_bytes(int n, int64_t blocks) {
  return decode_layout(n).fixed + static_cast<size_t>(blocks) * 192;
}

constexpr int kPlanThreads = 1024;

// one CTA: validation, status, and the exclusive scans that place each image in the workspace
__global__ void __launch_bounds__(kPlanThreads)
jpeg_plan_kernel(const Desc* __restrict__ descs, const int64_t* __restrict__ offsets,
                 const int64_t* __restrict__ rgb_offsets, int n, size_t ws_bytes, ImgPlan* __restrict__ plans,
                 int32_t* __restrict__ status) {
  typedef cub::BlockScan<long long, kPlanThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ long long carry_blocks, carry_iv;
  __shared__ int fits;
  for (int pass = 0; pass < 2; ++pass) {
    if (threadIdx.x == 0) {
      carry_blocks = 0;
      carry_iv = 0;
    }
    __syncthreads();
    for (int base = 0; base < n; base += kPlanThreads) {
      const int b = base + threadIdx.x;
      long long blocks = 0, iv = 0;
      bool ok = false;
      if (b < n) {
        const Desc& d = descs[b];
        const int64_t nbytes = offsets[b + 1] - offsets[b];
        ok = desc_ok(d) && offsets[b] >= 0 && d.scan_end <= nbytes &&
             rgb_offsets[b] >= 0 && rgb_offsets[b + 1] - rgb_offsets[b] >= static_cast<int64_t>(d.width) * d.height * 3;
        if (ok) {
          blocks = image_blocks(d);
          iv = d.n_intervals;
        }
      }
      long long eb, ei, tb, ti;
      Scan(tmp).ExclusiveSum(blocks, eb, tb);
      __syncthreads();
      Scan(tmp).ExclusiveSum(iv, ei, ti);
      __syncthreads();
      if (pass == 1 && b < n) {
        ImgPlan p;
        p.coef = (carry_blocks + eb) * 64;             // int16 elements in the coefficient region
        p.plane = (carry_blocks + eb) * 64;            // bytes in the plane region
        p.iv0 = carry_iv + ei;
        p.ok = ok && fits;
        p.pad = 0;
        plans[b] = p;
        status[b] = ok ? (fits ? 0 : kWorkspace) : kBadDesc;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        carry_blocks += tb;
        carry_iv += ti;
      }
      __syncthreads();
    }
    if (pass == 0 && threadIdx.x == 0) fits = decode_ws_bytes(n, carry_blocks) <= ws_bytes;
    __syncthreads();
  }
}

// libjpeg's jpeg_make_d_derived_tbl (maxcode, valoffset) and the lookahead, from the raw BITS / HUFFVAL
__host__ __device__ inline void build_huff_table(const uint8_t* bits, const uint8_t* vals, HuffTab& t) {
  int p = 0;
  int32_t code = 0;
  for (int l = 1; l <= 16; ++l) {
    const int cnt = bits[l - 1];
    t.valoff[l] = p - code;
    code += cnt;
    p += cnt;
    t.maxcode[l] = cnt ? code - 1 : -1;
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  for (int i = 0; i < 256; ++i) t.vals[i] = vals[i];
  for (int i = 0; i < (1 << kLookBits); ++i) {
    uint16_t e = 0;
    for (int l = 1; l <= kLookBits; ++l) {
      const int32_t c = i >> (kLookBits - l);
      if (c <= t.maxcode[l]) {                        // ascending lengths: a shorter code would have matched
        e = static_cast<uint16_t>((l << 8) | vals[c + t.valoff[l]]);
        break;
      }
    }
    t.look[i] = e;
  }
}

// one CTA per image, one warp per (class, table) slot the scan uses
__global__ void __launch_bounds__(256)
jpeg_tables_kernel(const Desc* __restrict__ descs, const ImgPlan* __restrict__ plans, HuffTab* __restrict__ tabs) {
  const int b = blockIdx.x;
  if (!plans[b].ok) return;
  const Desc& d = descs[b];
  const int w = threadIdx.x >> 5;
  const int cls = w >> 2, id = w & 3;
  bool used = false;
  for (int c = 0; c < d.ncomp; ++c) used |= (cls == 0 ? d.comp_td[c] : d.comp_ta[c]) == id;
  if (used && (threadIdx.x & 31) == 0) build_huff_table(d.huff_bits[cls][id], d.huff_vals[cls][id], tabs[static_cast<int64_t>(b) * 8 + w]);
}

// ---------------------------------------------------------------------------------------------- entropy decode
#ifdef __CUDA_ARCH__
#define LDG(p) __ldg(p)
#else
#define LDG(p) (*(p))
#endif

// Bit reader over [pos, stop) of one image: 0xFF00 -> 0xFF, any other 0xFF (after fill 0xFFs) ends the data, after
// which zeros are shifted in.  `real` counts the bits that came from data bytes.
struct BitReader {
  const uint8_t* p;
  int64_t pos, stop;
  uint64_t buf;
  int nbits;
  bool eod;
  int64_t real, used;

  __host__ __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t c = 0;
      if (!eod) {
        if (pos < stop) {
          c = LDG(p + pos);
          if (c == 0xFF) {
            int64_t q = pos + 1;
            while (q < stop && LDG(p + q) == 0xFF) ++q;
            if (q < stop && LDG(p + q) == 0) {
              pos = q + 1;
            } else {
              eod = true;
              c = 0;
            }
          } else {
            ++pos;
          }
          if (!eod) real += 8;
        } else {
          eod = true;
        }
      }
      buf |= static_cast<uint64_t>(c) << (56 - nbits);
      nbits += 8;
    }
  }
  __host__ __device__ __forceinline__ uint32_t peek16() const { return static_cast<uint32_t>(buf >> 48); }
  __host__ __device__ __forceinline__ void skip(int s) {
    buf <<= s;
    nbits -= s;
    used += s;
  }
  __host__ __device__ __forceinline__ uint32_t bits(int s) {          // 1 <= s <= 16
    const uint32_t r = static_cast<uint32_t>(buf >> (64 - s));
    skip(s);
    return r;
  }
};

// one symbol; -1: no such code
__host__ __device__ __forceinline__ int huff_decode(BitReader& br, const HuffTab& t) {
  const uint32_t look = br.peek16();
  const uint32_t e = t.look[look >> (16 - kLookBits)];
  if (e) {
    br.skip(e >> 8);
    return e & 0xFF;
  }
  for (int l = kLookBits + 1; l <= 16; ++l) {
    const int32_t code = static_cast<int32_t>(look >> (16 - l));
    if (code <= t.maxcode[l]) {
      br.skip(l);
      return t.vals[(code + t.valoff[l]) & 0xFF];
    }
  }
  return -1;
}

__host__ __device__ __forceinline__ int huff_extend(uint32_t r, int s) {
  return static_cast<int>(r) < (1 << (s - 1)) ? static_cast<int>(r) + static_cast<int>((~0u << s) + 1u) : static_cast<int>(r);
}

// Restart interval k of one image: its MCUs' blocks, zero-filled then written coefficient by coefficient
// (natural order).  img: the image's bytes; coef: its coefficients; iv: its interval table.  Returns 0 or a status bit.
__host__ __device__ inline int decode_interval(const uint8_t* img, const Desc& d, const HuffTab* T, int16_t* coef,
                                               const int32_t* iv, int k) {
  const int n_iv = d.n_intervals;
  const int32_t start = iv[k];
  const int32_t stop = k + 1 < n_iv ? iv[k + 1] : d.scan_end;
  if (start < d.scan_begin || start > stop || stop > d.scan_end) return kBadDesc;
  const int ncomp = d.ncomp;
  int16_t* cbase[3];
  int bw[3];
  int64_t acc = 0;
  for (int c = 0; c < ncomp; ++c) {
    cbase[c] = coef + acc;
    bw[c] = comp_blocks_w(d, c);
    acc += static_cast<int64_t>(bw[c]) * comp_blocks_h(d, c) * 64;
  }
  BitReader br;
  br.p = img;
  br.pos = start;
  br.stop = stop;
  br.buf = 0;
  br.nbits = 0;
  br.eod = false;
  br.real = 0;
  br.used = 0;
  const int64_t mcus = static_cast<int64_t>(d.mcus_x) * d.mcus_y;
  const int64_t m0 = d.restart_interval ? static_cast<int64_t>(k) * d.restart_interval : 0;
  int64_t m1 = d.restart_interval ? m0 + d.restart_interval : mcus;
  if (m1 > mcus) m1 = mcus;
  int pred[3] = {0, 0, 0};
  for (int64_t m = m0; m < m1; ++m) {
    const int my = static_cast<int>(m / d.mcus_x), mx = static_cast<int>(m - static_cast<int64_t>(my) * d.mcus_x);
    for (int c = 0; c < ncomp; ++c) {
      const int hh = c == 0 ? d.hmax : 1, vv = c == 0 ? d.vmax : 1;
      const HuffTab& dt = T[d.comp_td[c]];
      const HuffTab& at = T[4 + d.comp_ta[c]];
      for (int v = 0; v < vv; ++v)
        for (int h = 0; h < hh; ++h) {
          int16_t* blk = cbase[c] + (static_cast<int64_t>(my * vv + v) * bw[c] + mx * hh + h) * 64;
          for (int i = 0; i < 8; ++i) reinterpret_cast<int4*>(blk)[i] = make_int4(0, 0, 0, 0);
          br.fill();
          int s = huff_decode(br, dt);
          if (s < 0) return kBadCode;
          const int diff = s ? huff_extend(br.bits(s), s) : 0;
          pred[c] = static_cast<int>(static_cast<unsigned>(pred[c]) + static_cast<unsigned>(diff));
          blk[0] = static_cast<int16_t>(pred[c]);
          for (int kk = 1; kk < 64; ++kk) {
            br.fill();
            const int rs = huff_decode(br, at);
            if (rs < 0) return kBadCode;
            const int r = rs >> 4;
            s = rs & 15;
            if (s) {
              kk += r;
              const uint32_t v = br.bits(s);
              if (kk > 63) return kTooMany;
              blk[kNaturalAt(kk)] = static_cast<int16_t>(huff_extend(v, s));
            } else {
              if (r != 15) break;
              kk += 15;
            }
          }
        }
    }
    if (br.eod && br.used > br.real) return kOverrun;
  }
  return 0;
}

constexpr int kEntropyGx = 4;      // CTAs (of one warp) per image in x

// interval k of image b is run by CTA (k % kEntropyGx, b), lane (k / kEntropyGx) % 32: images without restart markers
// get one thread in a warp of their own
__global__ void __launch_bounds__(32)
jpeg_entropy_kernel(const uint8_t* __restrict__ data, const int64_t* __restrict__ offsets, const Desc* __restrict__ descs,
                    const int32_t* __restrict__ intervals, const ImgPlan* __restrict__ plans,
                    const HuffTab* __restrict__ tabs, int16_t* __restrict__ coef, int32_t* __restrict__ status) {
  const int b = blockIdx.y;
  const ImgPlan plan = plans[b];
  if (!plan.ok) return;
  const Desc& d = descs[b];
  for (int k = blockIdx.x + kEntropyGx * static_cast<int>(threadIdx.x); k < d.n_intervals; k += kEntropyGx * 32) {
    const int flag = decode_interval(data + offsets[b], d, tabs + static_cast<int64_t>(b) * 8, coef + plan.coef,
                                     intervals + plan.iv0, k);
    if (flag) atomicOr(status + b, flag);
  }
}

// ---------------------------------------------------------------------------------------------- IDCT
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int32_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// jidctint.c's post-IDCT range limit: index (x & 0x3FF) of the table that starts at sample_range_limit + CENTERJSAMPLE
__host__ __device__ __forceinline__ uint8_t idct_limit(int32_t v) {
  const int x = v & 0x3FF;
  if (x < 128) return static_cast<uint8_t>(x + 128);
  if (x < 512) return 255;
  if (x < 896) return 0;
  return static_cast<uint8_t>(x - 896);
}

// one 1-D pass of jpeg_idct_islow on in[0..7] (stride-free), results before the final descale
__host__ __device__ __forceinline__ void islow_1d(const int32_t in[8], int32_t out[8], int shift, int32_t add) {
  int32_t z2 = in[2], z3 = in[6];
  int32_t z1 = (z2 + z3) * F0541;
  int32_t tmp2 = z1 + z3 * (-F1847);
  int32_t tmp3 = z1 + z2 * F0765;
  z2 = in[0];
  z3 = in[4];
  int32_t tmp0 = static_cast<int32_t>(static_cast<uint32_t>(z2 + z3) << kConstBits);
  int32_t tmp1 = static_cast<int32_t>(static_cast<uint32_t>(z2 - z3) << kConstBits);
  const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int32_t z4 = tmp1 + tmp3;
  const int32_t z5 = (z3 + z4) * F1175;
  tmp0 = tmp0 * F0298;
  tmp1 = tmp1 * F2053;
  tmp2 = tmp2 * F3072;
  tmp3 = tmp3 * F1501;
  z1 = z1 * (-F0899);
  z2 = z2 * (-F2562);
  z3 = z3 * (-F1961);
  z4 = z4 * (-F0390);
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = (tmp10 + tmp3 + add) >> shift;
  out[7] = (tmp10 - tmp3 + add) >> shift;
  out[1] = (tmp11 + tmp2 + add) >> shift;
  out[6] = (tmp11 - tmp2 + add) >> shift;
  out[2] = (tmp12 + tmp1 + add) >> shift;
  out[5] = (tmp12 - tmp1 + add) >> shift;
  out[3] = (tmp13 + tmp0 + add) >> shift;
  out[4] = (tmp13 - tmp0 + add) >> shift;
}

// Range in which every IDCT of libjpeg-turbo gives jidctint.c's 32-bit C result.  Its x86-64 SIMD islow dequantises
// and adds pairs of values in 16-bit lanes, saturates (packssdw) the pass-1 results, and saturates its output where the
// C range limit wraps (index & 0x3FF).  The coefficients of an 8-bit image's blocks stay far inside this range.
constexpr int32_t kIdctInMax = 16383;        // |dequantised value|: a sum of two fits in int16
constexpr int32_t kIdctMidMax = 16383;       // |pass-1 result|: likewise
constexpr int32_t kIdctOutMin = -512, kIdctOutMax = 511;   // pass-2 result: C's wrapped index equals saturation

__host__ __device__ __forceinline__ bool outside(int32_t v, int32_t lo, int32_t hi) {
  return static_cast<uint32_t>(v - lo) > static_cast<uint32_t>(hi - lo);
}

// jpeg_idct_islow of one block: coefficients natural order, quant natural order -> 8 x 8 samples (row stride `ld`).
// Returns false when a value leaves the range above: libjpeg-turbo's SIMD and C IDCTs may then disagree (the C code's
// zero-AC shortcuts too: they equal the full pass only while the << CONST_BITS of the full pass does not overflow,
// which the range keeps), so the block's pixels are not Pillow's.
__host__ __device__ __forceinline__ bool idct_islow(const int16_t* co, const uint16_t* q, uint8_t* out, int64_t ld) {
  int32_t ws[64];
  bool bad = false;
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    int32_t in[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      in[r] = static_cast<int32_t>(co[r * 8 + col]) * static_cast<int32_t>(static_cast<int16_t>(q[r * 8 + col]));
      bad |= outside(in[r], -kIdctInMax, kIdctInMax);
    }
    islow_1d(in, o, kConstBits - kPass1Bits, 1 << (kConstBits - kPass1Bits - 1));
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      ws[r * 8 + col] = o[r];
      bad |= outside(o[r], -kIdctMidMax, kIdctMidMax);
    }
  }
  constexpr int kShift2 = kConstBits + kPass1Bits + 3;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    int32_t o[8];
    islow_1d(ws + r * 8, o, kShift2, 1 << (kShift2 - 1));
    uint8_t* dst = out + r * ld;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      dst[c] = idct_limit(o[c]);
      bad |= outside(o[c], kIdctOutMin, kIdctOutMax);
    }
  }
  return !bad;
}

constexpr int kIdctGx = 64;

__global__ void __launch_bounds__(128)
jpeg_idct_kernel(const Desc* __restrict__ descs, const ImgPlan* __restrict__ plans, const int16_t* __restrict__ coef,
                 uint8_t* __restrict__ planes, int32_t* __restrict__ status) {
  const int b = blockIdx.y;
  const ImgPlan plan = plans[b];
  if (!plan.ok) return;
  const Desc& d = descs[b];
  const int64_t total = image_blocks(d);
  for (int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; j < total;
       j += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int c = 0;
    int64_t r = j, first = 0;
    for (; c < d.ncomp - 1; ++c) {
      const int64_t nb = static_cast<int64_t>(comp_blocks_w(d, c)) * comp_blocks_h(d, c);
      if (r < nb) break;
      r -= nb;
      first += nb;
    }
    const int bwc = comp_blocks_w(d, c);
    const int by = static_cast<int>(r / bwc), bx = static_cast<int>(r - static_cast<int64_t>(by) * bwc);
    __align__(16) int16_t co[64];
    __align__(16) uint16_t q[64];
    const int4* src = reinterpret_cast<const int4*>(coef + plan.coef + j * 64);   // 128-byte aligned blocks
    // the descriptor guarantees 4-byte alignment only (an array of them has a 2792-byte stride)
    const uint32_t* qs = reinterpret_cast<const uint32_t*>(d.qt[d.comp_tq[c]]);
#pragma unroll
    for (int i = 0; i < 8; ++i) reinterpret_cast<int4*>(co)[i] = src[i];
#pragma unroll
    for (int i = 0; i < 32; ++i) reinterpret_cast<uint32_t*>(q)[i] = qs[i];
    const int64_t ld = static_cast<int64_t>(bwc) * 8;
    uint8_t* dst = planes + (plan.plane + first * 64) + (static_cast<int64_t>(by) * 8) * ld + bx * 8;
    if (!idct_islow(co, q, dst, ld)) atomicOr(status + b, kIdctRange);
  }
}

// ---------------------------------------------------------------------------------------------- upsample + colour
__host__ __device__ __forceinline__ uint8_t clamp255(int v) { return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// jdsample.c h2v1_fancy_upsample for output column x of a row `in` of cw >= 3 samples
__host__ __device__ __forceinline__ int fancy_h2v1(const uint8_t* in, int cw, int x) {
  const int i = x >> 1;
  const int v = in[i];
  if ((x & 1) == 0) return i == 0 ? v : (v * 3 + in[i - 1] + 1) >> 2;
  return i == cw - 1 ? v : (v * 3 + in[i + 1] + 2) >> 2;
}

// jdsample.c h2v2_fancy_upsample: `near` / `far` are the nearer and the further chroma row
__host__ __device__ __forceinline__ int fancy_h2v2(const uint8_t* near, const uint8_t* far, int cw, int x) {
  const int i = x >> 1;
  const int cs = near[i] * 3 + far[i];
  if ((x & 1) == 0) {
    if (i == 0) return (cs * 4 + 8) >> 4;
    return (cs * 3 + (near[i - 1] * 3 + far[i - 1]) + 8) >> 4;
  }
  if (i == cw - 1) return (cs * 4 + 7) >> 4;
  return (cs * 3 + (near[i + 1] * 3 + far[i + 1]) + 7) >> 4;
}

// one output pixel from the component planes (plane row strides pw[c])
__host__ __device__ __forceinline__ void jpeg_pixel(const Desc& d, const uint8_t* const pl[3], const int64_t pw[3], int y,
                                                    int x, uint8_t rgb[3]) {
  const int Y = pl[0][y * pw[0] + x];
  if (d.ncomp == 1) {
    rgb[0] = rgb[1] = rgb[2] = static_cast<uint8_t>(Y);
    return;
  }
  int ch[2];
  const int cw = (d.width + d.hmax - 1) / d.hmax, chh = (d.height + d.vmax - 1) / d.vmax;
  for (int k = 0; k < 2; ++k) {
    const uint8_t* p = pl[1 + k];
    if (d.hmax == 1) {
      ch[k] = p[y * pw[1 + k] + x];
    } else if (cw <= 2) {                                 // plain replication (downsampled_width <= 2)
      ch[k] = p[(y / d.vmax) * pw[1 + k] + (x >> 1)];
    } else if (d.vmax == 1) {
      ch[k] = fancy_h2v1(p + y * pw[1 + k], cw, x);
    } else {
      const int r = y >> 1;
      int o = (y & 1) ? r + 1 : r - 1;                    // context row: the edge row repeated outside the image
      o = o < 0 ? 0 : (o > chh - 1 ? chh - 1 : o);
      ch[k] = fancy_h2v2(p + r * pw[1 + k], p + o * pw[1 + k], cw, x);
    }
  }
  const int cb = ch[0] - 128, cr = ch[1] - 128;
  // jdcolor.c build_ycc_rgb_table, SCALEBITS 16: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802,
  // FIX(0.34414) = 22554, ONE_HALF = 1 << 15
  const int crr = (91881 * cr + 32768) >> 16;
  const int cbb = (116130 * cb + 32768) >> 16;
  const int g = ((-22554 * cb + 32768) + (-46802 * cr)) >> 16;
  rgb[0] = clamp255(Y + crr);
  rgb[1] = clamp255(Y + g);
  rgb[2] = clamp255(Y + cbb);
}

constexpr int kColourGx = 64;

__global__ void __launch_bounds__(256)
jpeg_colour_kernel(const Desc* __restrict__ descs, const ImgPlan* __restrict__ plans, const uint8_t* __restrict__ planes,
                   uint8_t* __restrict__ rgb_out, const int64_t* __restrict__ rgb_offsets) {
  const int b = blockIdx.y;
  const ImgPlan plan = plans[b];
  if (!plan.ok) return;
  const Desc& d = descs[b];
  const uint8_t* pl[3];
  int64_t pw[3];
  int64_t off = plan.plane;
  for (int c = 0; c < 3; ++c) {
    pl[c] = planes + off;
    pw[c] = c < d.ncomp ? static_cast<int64_t>(comp_blocks_w(d, c)) * 8 : 0;
    if (c < d.ncomp) off += pw[c] * comp_blocks_h(d, c) * 8;
  }
  uint8_t* out = rgb_out + rgb_offsets[b];
  const int64_t total = static_cast<int64_t>(d.width) * d.height;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / d.width), x = static_cast<int>(i - static_cast<int64_t>(y) * d.width);
    uint8_t rgb[3];
    jpeg_pixel(d, pl, pw, y, x, rgb);
    out[i * 3] = rgb[0];
    out[i * 3 + 1] = rgb[1];
    out[i * 3 + 2] = rgb[2];
  }
}

// ---------------------------------------------------------------------------------------------- Pillow bilinear resize
#ifdef __CUDA_ARCH__
#define DADD __dadd_rn
#define DSUB __dsub_rn
#define DMUL __dmul_rn
#define DDIV __ddiv_rn
#else
inline double DADD(double a, double b) { return a + b; }
inline double DSUB(double a, double b) { return a - b; }
inline double DMUL(double a, double b) { return a * b; }
inline double DDIV(double a, double b) { return a / b; }
#endif

// precompute_coeffs's kernel size: (int)ceil(support) * 2 + 1, support = filterscale (bilinear support 1)
__host__ __device__ inline int resize_ksize(int in_size, int out_size) {
  double scale = DDIV(static_cast<double>(in_size), static_cast<double>(out_size));
  if (scale < 1.0) scale = 1.0;
  return static_cast<int>(ceil(scale)) * 2 + 1;
}

// per image and axis: out_size entries of (xmin, count) then out_size * ksize int32 coefficients
__host__ __device__ inline int64_t resize_image_ints(int h, int w, int out_h, int out_w) {
  if (h < 1 || w < 1) return 0;
  return static_cast<int64_t>(out_w) * (2 + resize_ksize(w, out_w)) + static_cast<int64_t>(out_h) * (2 + resize_ksize(h, out_h));
}

struct ResizePlan {
  int64_t base;       // int32 offset of the image's coefficients
  int32_t ok, pad;
};

inline __host__ __device__ size_t resize_ws_bytes(int n, int64_t ints) {
  return align256(static_cast<size_t>(n) * sizeof(ResizePlan)) + static_cast<size_t>(ints) * 4;
}

__global__ void __launch_bounds__(kPlanThreads)
resize_plan_kernel(const int32_t* __restrict__ hw, int n, int out_h, int out_w, size_t ws_bytes,
                   ResizePlan* __restrict__ plans) {
  typedef cub::BlockScan<long long, kPlanThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ long long carry;
  __shared__ int fits;
  for (int pass = 0; pass < 2; ++pass) {
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += kPlanThreads) {
      const int b = base + threadIdx.x;
      const long long ints = b < n ? resize_image_ints(hw[2 * b], hw[2 * b + 1], out_h, out_w) : 0;
      long long e, t;
      Scan(tmp).ExclusiveSum(ints, e, t);
      __syncthreads();
      if (pass == 1 && b < n) {
        ResizePlan p;
        p.base = carry + e;
        p.ok = ints > 0 && fits;
        p.pad = 0;
        plans[b] = p;
      }
      __syncthreads();
      if (threadIdx.x == 0) carry += t;
      __syncthreads();
    }
    if (pass == 0 && threadIdx.x == 0) fits = resize_ws_bytes(n, carry) <= ws_bytes;
    __syncthreads();
  }
}

// Pillow's bilinear_filter((x - center + 0.5) * ss)
__host__ __device__ inline double bilinear_weight(int x, double center, double ss) {
  double t = DMUL(DADD(DSUB(static_cast<double>(x), center), 0.5), ss);
  if (t < 0.0) t = -t;
  return t < 1.0 ? DSUB(1.0, t) : 0.0;
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for output index xx of one axis
__host__ __device__ inline void resize_coeffs(int in_size, int out_size, int ksize, int xx, int32_t* bounds, int32_t* k) {
  const double scale = DDIV(static_cast<double>(in_size), static_cast<double>(out_size));
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = DMUL(1.0, filterscale);
  const double center = DMUL(DADD(static_cast<double>(xx), 0.5), scale);
  const double ss = DDIV(1.0, filterscale);
  int xmin = static_cast<int>(DADD(DSUB(center, support), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = static_cast<int>(DADD(DADD(center, support), 0.5));
  if (xmax > in_size) xmax = in_size;
  xmax -= xmin;
  if (xmax > ksize) xmax = ksize;                     // never taken: Pillow's window fits its own ksize
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x) ww = DADD(ww, bilinear_weight(x + xmin, center, ss));
  for (int x = 0; x < xmax; ++x) {
    double f = bilinear_weight(x + xmin, center, ss);
    if (ww != 0.0) f = DDIV(f, ww);
    k[x] = f < 0.0 ? static_cast<int32_t>(DADD(-0.5, DMUL(f, 4194304.0)))
                   : static_cast<int32_t>(DADD(0.5, DMUL(f, 4194304.0)));
  }
  for (int x = xmax; x < ksize; ++x) k[x] = 0;
  bounds[0] = xmin;
  bounds[1] = xmax;
}

constexpr int kResizeGx = 32;

__global__ void __launch_bounds__(256)
resize_coeff_kernel(const int32_t* __restrict__ hw, int out_h, int out_w, const ResizePlan* __restrict__ plans,
                    int32_t* __restrict__ ints) {
  const int b = blockIdx.y;
  const ResizePlan p = plans[b];
  if (!p.ok) return;
  const int h = hw[2 * b], w = hw[2 * b + 1];
  const int kx = resize_ksize(w, out_w), ky = resize_ksize(h, out_h);
  int32_t* xs = ints + p.base;                                    // [out_w][2] bounds, [out_w][kx] coefficients
  int32_t* ys = xs + static_cast<int64_t>(out_w) * (2 + kx);      // [out_h][2] bounds, [out_h][ky] coefficients
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < out_w + out_h; i += gridDim.x * blockDim.x) {
    if (i < out_w)
      resize_coeffs(w, out_w, kx, i, xs + 2 * i, xs + 2 * out_w + static_cast<int64_t>(i) * kx);
    else
      resize_coeffs(h, out_h, ky, i - out_w, ys + 2 * (i - out_w), ys + 2 * out_h + static_cast<int64_t>(i - out_w) * ky);
  }
}

__host__ __device__ __forceinline__ uint8_t clip8(int v) {
  if (v >= (1 << 30)) return 255;
  if (v <= 0) return 0;
  return static_cast<uint8_t>(v >> 22);
}

__global__ void __launch_bounds__(256)
resize_kernel(const uint8_t* __restrict__ in, const int64_t* __restrict__ in_offsets, const int32_t* __restrict__ hw,
              int out_h, int out_w, const ResizePlan* __restrict__ plans, const int32_t* __restrict__ ints,
              uint8_t* __restrict__ out) {
  const int b = blockIdx.y;
  const ResizePlan p = plans[b];
  uint8_t* o = out + static_cast<int64_t>(b) * out_h * out_w * 3;
  const int64_t total = static_cast<int64_t>(out_h) * out_w;
  const int h = hw[2 * b], w = hw[2 * b + 1];
  const int kx = p.ok ? resize_ksize(w, out_w) : 0, ky = p.ok ? resize_ksize(h, out_h) : 0;
  const int32_t* xs = ints + p.base;
  const int32_t* ys = xs + static_cast<int64_t>(out_w) * (2 + kx);
  const uint8_t* src = in + (p.ok ? in_offsets[b] : 0);
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (!p.ok) {
      o[i * 3] = o[i * 3 + 1] = o[i * 3 + 2] = 0;
      continue;
    }
    const int y = static_cast<int>(i / out_w), x = static_cast<int>(i - static_cast<int64_t>(y) * out_w);
    const int xmin = xs[2 * x], xn = xs[2 * x + 1];
    const int ymin = ys[2 * y], yn = ys[2 * y + 1];
    const int32_t* kxp = xs + 2 * out_w + static_cast<int64_t>(x) * kx;
    const int32_t* kyp = ys + 2 * out_h + static_cast<int64_t>(y) * ky;
    int acc0 = 1 << 21, acc1 = 1 << 21, acc2 = 1 << 21;
    for (int ty = 0; ty < yn; ++ty) {
      const uint8_t* row = src + (static_cast<int64_t>(ymin + ty) * w + xmin) * 3;
      int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
      for (int tx = 0; tx < xn; ++tx) {
        const int k = kxp[tx];
        s0 += row[tx * 3] * k;
        s1 += row[tx * 3 + 1] * k;
        s2 += row[tx * 3 + 2] * k;
      }
      const int k = kyp[ty];
      acc0 += clip8(s0) * k;
      acc1 += clip8(s1) * k;
      acc2 += clip8(s2) * k;
    }
    o[i * 3] = clip8(acc0);
    o[i * 3 + 1] = clip8(acc1);
    o[i * 3 + 2] = clip8(acc2);
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------- host parser
namespace {

inline int parse_fail(int rc, const char* what) {
  set_error("jpeg_parse: %s", what);
  return rc;
}

inline int rd16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

int jpeg_parse(const uint8_t* d, int64_t n, Desc* D, int32_t* iv, int64_t cap) {
  memset(D, 0, sizeof(*D));
  if (n < 2) return parse_fail(DIRB200_JPEG_MALFORMED, "fewer than 2 bytes");
  if (d[0] != 0xFF || d[1] != 0xD8) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "not a JPEG (no SOI)");
  bool jfif = false, adobe = false, sof = false;
  int adobe_transform = 0;
  bool have_q[4] = {false, false, false, false};
  bool have_h[2][4] = {{false, false, false, false}, {false, false, false, false}};
  int comp_id[3] = {0, 0, 0};
  int64_t pos = 2;
  for (;;) {
    // a marker: 0xFF, any fill 0xFFs, the code
    if (pos >= n) return parse_fail(DIRB200_JPEG_MALFORMED, "no SOS before the end of the data");
    if (d[pos] != 0xFF) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "bytes between markers");
    while (pos < n && d[pos] == 0xFF) ++pos;
    if (pos >= n) return parse_fail(DIRB200_JPEG_MALFORMED, "truncated marker");
    const int m = d[pos++];
    if (m == 0xD8 || m == 0xD9 || m == 0x00) return parse_fail(DIRB200_JPEG_MALFORMED, "SOI / EOI / 0 before SOS");
    if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "RST / TEM outside a scan");
    if (pos + 2 > n) return parse_fail(DIRB200_JPEG_MALFORMED, "truncated marker length");
    const int len = rd16(d + pos);
    if (len < 2) return parse_fail(DIRB200_JPEG_MALFORMED, "marker length below 2");
    if (pos + len > n) return parse_fail(DIRB200_JPEG_MALFORMED, "marker segment runs past the data");
    const uint8_t* s = d + pos + 2;
    const int sl = len - 2;
    const int64_t next = pos + len;
    if (m == 0xE0) {
      if (sl >= 14 && s[0] == 'J' && s[1] == 'F' && s[2] == 'I' && s[3] == 'F' && s[4] == 0) jfif = true;
    } else if (m == 0xEE) {
      if (sl >= 12 && s[0] == 'A' && s[1] == 'd' && s[2] == 'o' && s[3] == 'b' && s[4] == 'e') {
        adobe = true;
        adobe_transform = s[11];
      }
    } else if (m == 0xDB) {                                              // DQT
      int q = 0;
      while (q < sl) {
        const int pq = s[q] >> 4, tq = s[q] & 15;
        if (tq > 3) return parse_fail(DIRB200_JPEG_MALFORMED, "DQT table index above 3");
        if (pq > 1) return parse_fail(DIRB200_JPEG_MALFORMED, "DQT precision above 1");
        const int need = 1 + 64 * (pq + 1);
        if (q + need > sl) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "short DQT table");
        for (int k = 0; k < 64; ++k) {
          const int v = pq ? rd16(s + q + 1 + 2 * k) : s[q + 1 + k];
          if (v > 32767) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "DQT value above 32767");
          D->qt[tq][kNatural[k]] = static_cast<uint16_t>(v);
        }
        have_q[tq] = true;
        q += need;
      }
    } else if (m == 0xC4) {                                              // DHT
      int q = 0;
      while (q < sl) {
        if (q + 17 > sl) return parse_fail(DIRB200_JPEG_MALFORMED, "short DHT");
        const int tc = s[q] >> 4, th = s[q] & 15;
        if (tc > 1 || th > 3) return parse_fail(DIRB200_JPEG_MALFORMED, "DHT table index");
        int count = 0;
        for (int l = 0; l < 16; ++l) count += s[q + 1 + l];
        if (count > 256 || q + 17 + count > sl) return parse_fail(DIRB200_JPEG_MALFORMED, "bad DHT symbol count");
        memcpy(D->huff_bits[tc][th], s + q + 1, 16);
        memset(D->huff_vals[tc][th], 0, 256);
        memcpy(D->huff_vals[tc][th], s + q + 17, count);
        have_h[tc][th] = true;
        q += 17 + count;
      }
    } else if (m == 0xDD) {                                              // DRI
      if (sl != 2) return parse_fail(DIRB200_JPEG_MALFORMED, "DRI length");
      D->restart_interval = rd16(s);
    } else if (m == 0xC0 || m == 0xC1) {                                 // SOF0 / SOF1
      if (sof) return parse_fail(DIRB200_JPEG_MALFORMED, "second SOF");
      sof = true;
      if (sl < 6) return parse_fail(DIRB200_JPEG_MALFORMED, "short SOF");
      if (s[0] != 8) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "sample precision other than 8");
      D->height = rd16(s + 1);
      D->width = rd16(s + 3);
      const int nf = s[5];
      if (sl != 6 + 3 * nf) return parse_fail(DIRB200_JPEG_MALFORMED, "SOF length");
      if (D->width == 0 || nf == 0) return parse_fail(DIRB200_JPEG_MALFORMED, "empty image");
      if (D->height == 0) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "height from a DNL marker");
      if (nf != 1 && nf != 3) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "component count other than 1 or 3");
      D->ncomp = nf;
      for (int c = 0; c < nf; ++c) {
        comp_id[c] = s[6 + 3 * c];
        D->comp_h[c] = s[7 + 3 * c] >> 4;
        D->comp_v[c] = s[7 + 3 * c] & 15;
        D->comp_tq[c] = s[8 + 3 * c];
        if (D->comp_h[c] < 1 || D->comp_h[c] > 4 || D->comp_v[c] < 1 || D->comp_v[c] > 4 || D->comp_tq[c] > 3)
          return parse_fail(DIRB200_JPEG_MALFORMED, "bad sampling factor or quantisation table index");
      }
    } else if ((m >= 0xC2 && m <= 0xCF) || m == 0xDE || m == 0xDF) {   // other SOFn, DAC, DHP, EXP
      return parse_fail(DIRB200_JPEG_UNSUPPORTED, "progressive, lossless, hierarchical or arithmetic coding");
    } else if (m == 0xDA) {                                              // SOS
      if (!sof) return parse_fail(DIRB200_JPEG_MALFORMED, "SOS before SOF");
      if (sl < 1) return parse_fail(DIRB200_JPEG_MALFORMED, "short SOS");
      const int ns = s[0];
      if (sl != 4 + 2 * ns) return parse_fail(DIRB200_JPEG_MALFORMED, "SOS length");
      if (ns != D->ncomp) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "a scan without every component");
      for (int c = 0; c < ns; ++c) {
        if (s[1 + 2 * c] != comp_id[c]) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "scan components out of frame order");
        D->comp_td[c] = s[2 + 2 * c] >> 4;
        D->comp_ta[c] = s[2 + 2 * c] & 15;
        if (D->comp_td[c] > 3 || D->comp_ta[c] > 3) return parse_fail(DIRB200_JPEG_MALFORMED, "Huffman table index");
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0)
        return parse_fail(DIRB200_JPEG_UNSUPPORTED, "spectral selection / approximation of a non-sequential scan");
      // colour space (libjpeg's default_decompress_parms) and sampling
      if (D->ncomp == 3) {
        bool rgb;
        if (jfif) rgb = false;
        else if (adobe) rgb = adobe_transform == 0;
        else rgb = comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B';
        if (rgb) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "RGB-coded (untransformed) colour");
        const int h = D->comp_h[0], v = D->comp_v[0];
        if (!((h == 1 && v == 1) || (h == 2 && v == 1) || (h == 2 && v == 2)) || D->comp_h[1] != 1 ||
            D->comp_v[1] != 1 || D->comp_h[2] != 1 || D->comp_v[2] != 1)
          return parse_fail(DIRB200_JPEG_UNSUPPORTED, "sampling other than 4:4:4, 4:2:2 or 4:2:0");
        D->hmax = h;
        D->vmax = v;
      } else {
        if (D->comp_h[0] != 1 || D->comp_v[0] != 1) return parse_fail(DIRB200_JPEG_UNSUPPORTED, "grayscale sampling");
        D->hmax = D->vmax = 1;
      }
      if (static_cast<int64_t>(D->width) * D->height > kMaxPixels)
        return parse_fail(DIRB200_JPEG_UNSUPPORTED, "more than 2^26 pixels");
      for (int c = 0; c < D->ncomp; ++c) {
        if (!have_q[D->comp_tq[c]]) return parse_fail(DIRB200_JPEG_MALFORMED, "undefined quantisation table");
        if (!have_h[0][D->comp_td[c]] || !have_h[1][D->comp_ta[c]])
          return parse_fail(DIRB200_JPEG_UNSUPPORTED, "undefined Huffman table");
        if (!huff_table_ok(D->huff_bits[0][D->comp_td[c]], D->huff_vals[0][D->comp_td[c]], true) ||
            !huff_table_ok(D->huff_bits[1][D->comp_ta[c]], D->huff_vals[1][D->comp_ta[c]], false))
          return parse_fail(DIRB200_JPEG_MALFORMED, "bad Huffman table");
      }
      D->mcus_x = (D->width + 8 * D->hmax - 1) / (8 * D->hmax);
      D->mcus_y = (D->height + 8 * D->vmax - 1) / (8 * D->vmax);
      const int64_t mcus = static_cast<int64_t>(D->mcus_x) * D->mcus_y;
      const int64_t n_iv = D->restart_interval ? (mcus + D->restart_interval - 1) / D->restart_interval : 1;
      if (n_iv > (n + 3) / 2) return parse_fail(DIRB200_JPEG_MALFORMED, "more restart intervals than the data can hold");
      if (n_iv > cap) return parse_fail(DIRB200_ERR_ARG, "interval table too small");
      D->n_intervals = static_cast<int32_t>(n_iv);
      // the entropy-coded segment: stuffed 0xFF00, RSTn in sequence, up to the first other marker
      int64_t p = next;
      D->scan_begin = static_cast<int32_t>(p);
      iv[0] = static_cast<int32_t>(p);
      int64_t found = 1;
      int64_t end = -1, mpos = -1;
      while (end < 0) {
        const void* ff = p < n ? memchr(d + p, 0xFF, static_cast<size_t>(n - p)) : nullptr;
        if (ff == nullptr) return parse_fail(DIRB200_JPEG_MALFORMED, "entropy-coded data runs to the end of the file");
        const int64_t f = static_cast<const uint8_t*>(ff) - d;
        int64_t q = f + 1;
        while (q < n && d[q] == 0xFF) ++q;
        if (q >= n) return parse_fail(DIRB200_JPEG_MALFORMED, "entropy-coded data runs to the end of the file");
        if (d[q] == 0x00) {
          p = q + 1;
        } else if (d[q] >= 0xD0 && d[q] <= 0xD7) {
          if (found >= n_iv || d[q] != 0xD0 + ((found - 1) & 7))
            return parse_fail(DIRB200_JPEG_MALFORMED, "restart marker out of sequence");
          iv[found++] = static_cast<int32_t>(q + 1);
          p = q + 1;
        } else {
          end = f;
          mpos = q;
        }
      }
      if (found != n_iv) return parse_fail(DIRB200_JPEG_MALFORMED, "fewer restart markers than intervals");
      D->scan_end = static_cast<int32_t>(end);
      // after the scan: only EOI, or markers libjpeg skips, may follow
      pos = mpos;
      for (;;) {
        const int mm = d[pos++];
        if (mm == 0xD9) return 0;
        if (mm == 0xDA || mm == 0xDC || (mm >= 0xC0 && mm <= 0xCF && mm != 0xC4 && mm != 0xC8 && mm != 0xCC))
          return parse_fail(DIRB200_JPEG_UNSUPPORTED, "a second scan, DNL or SOF after the scan");
        if ((mm >= 0xD0 && mm <= 0xD8) || mm == 0x01 || mm == 0x00)
          return parse_fail(DIRB200_JPEG_UNSUPPORTED, "unexpected marker after the scan");
        if (pos + 2 > n) return parse_fail(DIRB200_JPEG_MALFORMED, "truncated after the scan");
        const int l2 = rd16(d + pos);
        if (l2 < 2 || pos + l2 > n) return parse_fail(DIRB200_JPEG_MALFORMED, "truncated after the scan");
        pos += l2;
        if (pos >= n || d[pos] != 0xFF) return parse_fail(DIRB200_JPEG_MALFORMED, "no EOI");
        while (pos < n && d[pos] == 0xFF) ++pos;
        if (pos >= n) return parse_fail(DIRB200_JPEG_MALFORMED, "no EOI");
      }
    } else if (m == 0xDC) {
      return parse_fail(DIRB200_JPEG_UNSUPPORTED, "DNL");
    } else if (!((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) {
      return parse_fail(DIRB200_JPEG_UNSUPPORTED, "unknown marker");
    }
    pos = next;
  }
}

}  // namespace

}  // namespace dirb200

using namespace dirb200;

extern "C" {

size_t dirb200_jpeg_desc_bytes(void) { return sizeof(dirb200_jpeg_desc); }

int dirb200_jpeg_parse(const uint8_t* data_host, int64_t nbytes, dirb200_jpeg_desc* desc_host, int32_t* intervals_host,
                       int64_t max_intervals) {
  DIRB_CHECK_ARG(desc_host && intervals_host && (data_host || nbytes == 0), "jpeg_parse: null pointer");
  DIRB_CHECK_ARG(nbytes >= 0 && nbytes < (int64_t(1) << 31), "jpeg_parse: nbytes %lld outside [0, 2^31)",
                 static_cast<long long>(nbytes));
  DIRB_CHECK_ARG(max_intervals >= 1, "jpeg_parse: max_intervals must be at least 1");
  return jpeg_parse(data_host, nbytes, desc_host, intervals_host, max_intervals);
}

size_t dirb200_jpeg_decode_workspace_bytes(const dirb200_jpeg_desc* descs_host, int n) {
  if (descs_host == nullptr || n <= 0) return 0;
  int64_t blocks = 0;
  for (int b = 0; b < n; ++b)
    if (desc_ok(descs_host[b])) blocks += image_blocks(descs_host[b]);
  return decode_ws_bytes(n, blocks);
}

int dirb200_jpeg_decode(const uint8_t* data, const int64_t* offsets, const dirb200_jpeg_desc* descs,
                        const int32_t* intervals, int n, uint8_t* rgb_out, const int64_t* rgb_offsets, int32_t* status,
                        void* workspace, size_t workspace_bytes, void* stream) {
  DIRB_CHECK_ARG(data && offsets && descs && intervals && rgb_out && rgb_offsets && status && workspace,
                 "jpeg_decode: null pointer");
  DIRB_CHECK_ARG(n >= 1 && n <= 65535, "jpeg_decode: n = %d outside [1, 65535]", n);
  const DecodeLayout L = decode_layout(n);
  DIRB_CHECK_ARG(workspace_bytes >= L.fixed, "jpeg_decode: workspace %zu bytes, needs at least %zu", workspace_bytes,
                 L.fixed);
  cudaStream_t st = as_stream(stream);
  char* ws = static_cast<char*>(workspace);
  ImgPlan* plans = reinterpret_cast<ImgPlan*>(ws + L.plans);
  HuffTab* tabs = reinterpret_cast<HuffTab*>(ws + L.tabs);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + L.coef);
  // planes follow the coefficients; the plan kernel checked that both fit, so the split point is only read there
  const size_t coef_cap = (workspace_bytes - L.fixed) / 192 * 128;
  uint8_t* planes = reinterpret_cast<uint8_t*>(ws + L.coef + coef_cap);
  jpeg_plan_kernel<<<1, kPlanThreads, 0, st>>>(descs, offsets, rgb_offsets, n, workspace_bytes, plans, status);
  DIRB_LAUNCHED();
  jpeg_tables_kernel<<<n, 256, 0, st>>>(descs, plans, tabs);
  DIRB_LAUNCHED();
  jpeg_entropy_kernel<<<dim3(kEntropyGx, n), 32, 0, st>>>(data, offsets, descs, intervals, plans, tabs, coef, status);
  DIRB_LAUNCHED();
  jpeg_idct_kernel<<<dim3(kIdctGx, n), 128, 0, st>>>(descs, plans, coef, planes, status);
  DIRB_LAUNCHED();
  jpeg_colour_kernel<<<dim3(kColourGx, n), 256, 0, st>>>(descs, plans, planes, rgb_out, rgb_offsets);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

size_t dirb200_resize_bilinear_workspace_bytes(const int32_t* hw_host, int n, int out_h, int out_w) {
  if (hw_host == nullptr || n <= 0 || out_h <= 0 || out_w <= 0) return 0;
  int64_t ints = 0;
  for (int b = 0; b < n; ++b) ints += resize_image_ints(hw_host[2 * b], hw_host[2 * b + 1], out_h, out_w);
  return resize_ws_bytes(n, ints);
}

int dirb200_resize_bilinear_u8(const uint8_t* in, const int64_t* in_offsets, const int32_t* hw, int n, int out_h,
                               int out_w, uint8_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  DIRB_CHECK_ARG(in && in_offsets && hw && out && workspace, "resize_bilinear_u8: null pointer");
  DIRB_CHECK_ARG(n >= 1 && n <= 65535, "resize_bilinear_u8: n = %d outside [1, 65535]", n);
  DIRB_CHECK_ARG(out_h >= 1 && out_w >= 1 && out_h <= 65535 && out_w <= 65535,
                 "resize_bilinear_u8: output size %d x %d", out_h, out_w);
  const size_t head = align256(static_cast<size_t>(n) * sizeof(ResizePlan));
  DIRB_CHECK_ARG(workspace_bytes >= head, "resize_bilinear_u8: workspace %zu bytes, needs at least %zu",
                 workspace_bytes, head);
  cudaStream_t st = as_stream(stream);
  ResizePlan* plans = static_cast<ResizePlan*>(workspace);
  int32_t* ints = reinterpret_cast<int32_t*>(static_cast<char*>(workspace) + head);
  resize_plan_kernel<<<1, kPlanThreads, 0, st>>>(hw, n, out_h, out_w, workspace_bytes, plans);
  DIRB_LAUNCHED();
  resize_coeff_kernel<<<dim3(4, n), 256, 0, st>>>(hw, out_h, out_w, plans, ints);
  DIRB_LAUNCHED();
  resize_kernel<<<dim3(kResizeGx, n), 256, 0, st>>>(in, in_offsets, hw, out_h, out_w, plans, ints, out);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

}  // extern "C"
