// Implicit-GEMM convolution on the Hopper tensor cores (wgmma + TMA + mbarrier),
// NHWC bf16 activations, fp32 accumulation.  Stage (i) of the hot path:
// replaces the cuDNN convolutions behind agedb-dir/resnet.py:46-51,79,112-118
// (forward) and their autograd backward (data and weight gradients).
//
// Persistent kernel: one CTA per SM walks the 128 x BN output tiles; the smem ring (full / empty mbarrier per stage)
// runs across tile boundaries.  Warpgroup 0 produces (cp.async gather of A + TMA of B, or TMA of both); warpgroups 1
// and 2 consume rows [0, 64) / [64, 128) of the tile with wgmma, accumulators in registers, epilogue from registers.
//
//   FPROP  Y[p, co]  = sum_k  A[p, k] W[co, k]      A, W K-major      (k = (r, s, c))
//   DGRAD  dX[p, c]  = sum_k  A'[p, k] Wt[c, k]     same kernel, transposed gather (k = (r, s, co))
//   WGRAD  dW[k, co] = sum_p  A[p, k] dY[p, co]     both operands MN-major, K = pixels, split-K partials
#include <stdlib.h>
#include "common.cuh"
#include "tc.cuh"
#include "conv.cuh"

namespace dirb200 {
using namespace tc;

constexpr int BM = 128;  // GEMM rows per tile (pixels; for wgrad: 2 chunks x 64 gathered channels)
constexpr int BK = 64;   // bf16 elements per k-block = one 128-byte swizzle row
constexpr int kProducerThreads = 128;   // warpgroup 0
constexpr int kThreads = 384;           // + two consumer warpgroups
constexpr int kMaxSmemBytes = 232448;   // opt-in shared memory per block (227 KB)

struct IgemmParams {
  const __nv_bfloat16* src;  // gathered tensor, NHWC
  int n, hs, ws, cs;         // its shape
  int hm, wm;                // pixel grid that indexes GEMM rows (fprop/wgrad: conv output grid; dgrad: conv input grid)
  int kh, kw, stride, pad;
  int transposed;            // 0: fprop-style gather, 1: dgrad-style (source = dY of a strided conv)
  // stride-2 dgrad runs as 4 launches, one per output-pixel parity class (py, px): rows index the class grid
  // (hm x wm), the real pixel is (2y'+py, 2x'+px) of the full_h x full_w image, and only the filter taps whose
  // parity matches (tap_list) are visited -- 9 tap-passes over quarter-size grids instead of 9 over the full one.
  int cls_on, cls_py, cls_px, full_h, full_w;
  int ntaps_c;               // taps visited by this launch
  int tap_list[kMaxTaps];    // their indices r*kw + s (identity when cls_on == 0)
  // per visited tap (index = position in tap_list), filled by finish_params(): element offset of the tap from the
  // row's origin in the gathered tensor, and the im2col-TMA offsets (flipped for dgrad)
  long long tap_eoff[kMaxTaps];
  unsigned short tap_r[kMaxTaps], tap_s[kMaxTaps];
  FastDiv fd_hw, fd_wm, fd_cpb, fd_kw, fd_ntiles, fd_persplit;
  int cpb;                   // 64-channel blocks per filter tap (cs / 64); stem: unused
  long long pixels;          // n * hm * wm
  int num_kblocks;           // fprop/dgrad: kh*kw*cpb ; wgrad: ceil(pixels / 64)
  int kblocks_per_split;     // wgrad split-K
  int total_chunks;          // wgrad: kh*kw*cpb (64-row chunks of the K_total x Cout result)
  int m_tiles, n_tiles;      // tiles along GEMM M / N
  int num_tiles;             // m_tiles * n_tiles * splits (persistent CTAs walk them round-robin)
  int a_mode;                // ATMA kernels: 1 = A is a plain [pixels][channels] matrix (tiled TMA), 2 = im2col TMA
  int i2c_stride, i2c_lo;    // im2col: base pixel of GEMM row (y, x) = (y * i2c_stride + i2c_lo, x * i2c_stride + i2c_lo)
  int ldc;                   // output row stride in elements (Cout for fprop, Cin for dgrad, Cout for wgrad partials)
  void* out;                 // bf16 [pixels][ldc]   or   fp32 [splits][Cout][total_chunks*64]
  // fprop only, optional: per-column sum / sum of squares of the (bf16-rounded) output = the BatchNorm batch
  // statistics of the layer, carried in per-warp shared-memory slots over all tiles of the CTA and written once per
  // CTA as stat_out[blockIdx.x][2][ldc] (fp32), columns [n_tile * BN, n_tile * BN + BN) of the CTA's fixed n_tile only
  // (see StatLayout for which rows hold which columns)
  float* stat_out;
  // AFFINE kernels (inference: BatchNorm folded into the conv epilogue, agedb-dir/train.py:286-335 / resnet.py:46-66 in
  // eval mode): out = [relu]( acc * epi_scale[col] + epi_shift[col] [+ epi_res[row][col]] )
  const float* epi_scale;
  const float* epi_shift;
  const __nv_bfloat16* epi_res;   // optional residual (identity / downsample branch), same [pixels][ldc] layout as out
  int epi_relu;
  // BSTAT kernels (stride-1 dgrad whose output dX is the gradient g w.r.t. a = relu(bn(y)) of the PREVIOUS layer): the
  // epilogue also accumulates that BatchNorm's backward moments  S0 = sum dz,  S1 = sum dz * y  with
  // dz = g * [y * bst_scale + bst_shift > 0]  (g as stored, bf16) into stat_out[CTA][2][ldc] -- the separate
  // bn_bwd_reduce pass over (g, y) disappears; y has the layout of the output ([pixels][ldc])
  const __nv_bfloat16* bst_y;
  const float* bst_scale;
  const float* bst_shift;
};

template <int BN, bool STAGED_EPI>
struct Cfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // as many ring stages as fit next to the epilogue buffers; one persistent CTA per SM
  static constexpr int kStages = BN == 128 ? (STAGED_EPI ? 5 : 6) : 8;
  static constexpr int kBarOffset = kStages * kStageBytes;
  // fprop / dgrad: a per-consumer-warp staging tile of 16 rows x BN bf16 (+16 B per row: conflict-free fragment writes)
  static constexpr int kStageRowBytes = BN * 2 + 16;
  static constexpr int kEpiWarpBytes = 16 * kStageRowBytes;
  static constexpr int kEpiOffset = kBarOffset + 256;           // after the mbarriers (2 * kStages * 8 <= 128 B)
  // per consumer warp: [2 (sum, sum of squares)][BN] fp32 running column sums of the BN statistics
  static constexpr int kStatWarpBytes = 2 * BN * 4;
  static constexpr int kStatOffset = kEpiOffset + (STAGED_EPI ? 8 * kEpiWarpBytes : 0);
  static constexpr int kSmemBytes = kStatOffset + (STAGED_EPI ? 8 * kStatWarpBytes : 0) + 1024;
  static_assert(kSmemBytes <= kMaxSmemBytes, "shared memory budget");
};

// ---- A-operand gather --------------------------------------------------------------------------------
// A tile row = 128 contiguous bytes of the source tensor (64 channels of one pixel; stem: 4 taps x 16 channels).
// The 8 lanes of a quarter-warp copy the 8 x 16 B of one row, so every warp-wide cp.async touches 4 full 128-byte
// lines (fully coalesced L2 requests); a thread therefore serves 8 different rows, always the same 16-byte column.
//
// packed pixel: bit 31 valid | n (13 bits) << 18 | y (9 bits) << 9 | x (9 bits)
__device__ __forceinline__ uint32_t pack_pixel(long long p, const IgemmParams& P) {
  if (p >= P.pixels) return 0u;
  uint32_t n, rem, y, x;
  P.fd_hw.divmod(static_cast<uint32_t>(p), n, rem);
  P.fd_wm.divmod(rem, y, x);
  return 0x80000000u | (n << 18) | (y << 9) | x;
}

// Row-invariant part of the gather address, unpacked once: image base row n*hs, and the tap-0 coordinates
// (fprop-style: y*stride - pad ; dgrad-style: y + pad).
struct RowPre {
  int nb, yb, xb;   // yb == INT_MIN/2 marks an invalid (out-of-range) row
};
__device__ __forceinline__ RowPre row_pre(const IgemmParams& P, uint32_t pk) {
  RowPre rp;
  const int n = (pk >> 18) & 0x1FFF;
  int y = (pk >> 9) & 0x1FF, x = pk & 0x1FF;
  if (P.cls_on) {
    y = 2 * y + P.cls_py;
    x = 2 * x + P.cls_px;
  }
  rp.nb = n * P.hs;
  if (!P.transposed) {
    rp.yb = y * P.stride - P.pad;
    rp.xb = x * P.stride - P.pad;
  } else {
    rp.yb = y + P.pad;
    rp.xb = x + P.pad;
  }
  if (!(pk >> 31)) rp.yb = -(1 << 28);
  return rp;
}

// Source of the 16 bytes at channel offset `coff` of filter tap (r, s).
// fprop-style: input pixel (y*stride - pad + r, x*stride - pad + s).
// dgrad-style: the conv-output pixel (ho, wo) with ho*stride - pad + r == y (stride 1 or 2; must divide exactly).
__device__ __forceinline__ const __nv_bfloat16* tap_source(const IgemmParams& P, const RowPre& rp, int r, int s,
                                                           int coff, bool& ok) {
  int hi, wi;
  ok = true;
  if (!P.transposed) {
    hi = rp.yb + r;
    wi = rp.xb + s;
  } else {
    hi = rp.yb - r;
    wi = rp.xb - s;
    if (P.stride == 2) {
      ok = ((hi | wi) & 1) == 0;
      hi >>= 1;
      wi >>= 1;
    }
  }
  ok = ok && static_cast<unsigned>(hi) < static_cast<unsigned>(P.hs) &&
       static_cast<unsigned>(wi) < static_cast<unsigned>(P.ws);
  return ok ? P.src + (static_cast<size_t>(rp.nb + hi) * P.ws + wi) * P.cs + coff : P.src;
}

// ATMA: the A operand comes by TMA -- tiled maps for 1x1 / stride-1 convolutions (a plain [pixels][channels] matrix:
// K-major 64 x 128 boxes for fprop / dgrad, two 64 x 64 MN-major boxes for wgrad), im2col-mode maps for the 3x3 and
// strided ones -- issued by warp 0.  Without ATMA (stem, or with the TMA forms switched off) warps 0-3 gather the rows
// with cp.async.
template <int BN, bool WGRAD, bool STEM, bool ATMA = false, bool AFFINE = false, bool BSTAT = false>
__global__ void __launch_bounds__(kThreads, 1)
igemm_kernel(const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_a,
             const IgemmParams P) {
  using C = Cfg<BN, !WGRAD>;
  static_assert(BN == 64 || BN == 128, "tile width: one m64n64 / m64n128 wgmma per warpgroup and k step");
  static_assert(!ATMA || !STEM, "TMA-fed A operand: not for the stem");
  // the folded-BN epilogue reads only the accumulators and P: it does not depend on how the A operand arrived
  static_assert(!AFFINE || (!WGRAD && !STEM), "folded-BN epilogue: non-stem fprop GEMMs only");
  static_assert(!BSTAT || (ATMA && !WGRAD && !AFFINE), "BN-backward moments in the epilogue: TMA-fed dgrad GEMMs only");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* const smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + C::kBarOffset;
  auto a_addr = [&](int s) { return smem_base + s * C::kStageBytes; };
  auto b_addr = [&](int s) { return smem_base + s * C::kStageBytes + C::kABytes; };
  constexpr uint32_t nstages = C::kStages;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::kStages + s); };
  const int warp = static_cast<int>(threadIdx.x >> 5), lane = threadIdx.x & 31;

  // Tile walk.  wgrad: work items t = (split, m_tile, n_tile) handed out round-robin (n fastest).
  // fprop / dgrad: every CTA keeps ONE n_tile for the whole launch -- CTA c owns n = c % n_tiles and walks
  // m = c / n_tiles, + G, + 2G, ... (G = CTAs sharing that n); neighbouring CTAs still work on the same A rows at the
  // same time (L2 reuse), and the epilogue can carry per-column sums (BN statistics) across all of its tiles and
  // flush them once.
  int tile_first, tile_end, tile_step, fixed_n = 0;
  if constexpr (WGRAD) {
    tile_first = blockIdx.x; tile_end = P.num_tiles; tile_step = gridDim.x;
  } else {
    uint32_t gi, nn;
    P.fd_ntiles.divmod(blockIdx.x, gi, nn);
    fixed_n = static_cast<int>(nn);
    tile_first = static_cast<int>(gi);
    tile_end = P.m_tiles;
    tile_step = static_cast<int>(P.fd_ntiles.div(gridDim.x - 1u - nn)) + 1;
  }
  auto decode_tile = [&](int t, int& split, int& m_tile, int& n_tile, int& kb_begin, int& nk) {
    if constexpr (WGRAD) {
      uint32_t sp, rem, mt, nt;
      P.fd_persplit.divmod(static_cast<uint32_t>(t), sp, rem);
      P.fd_ntiles.divmod(rem, mt, nt);
      split = static_cast<int>(sp);
      m_tile = static_cast<int>(mt);
      n_tile = static_cast<int>(nt);
      kb_begin = split * P.kblocks_per_split;
      const int kb_end = min(P.num_kblocks, kb_begin + P.kblocks_per_split);
      nk = max(0, kb_end - kb_begin);
    } else {
      split = 0;
      m_tile = t;
      n_tile = fixed_n;
      kb_begin = 0;
      nk = P.num_kblocks;
    }
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::kStages; ++s) {
      // TMA-fed: the TMA thread's one expect_tx arrival; gather-fed: + the 128 gather threads
      mbar_init(full_bar(s), ATMA ? 1 : kProducerThreads + 1);
      mbar_init(empty_bar(s), 8);          // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    if constexpr (!ATMA) {
      // ===== A producer (4 warps) + B by TMA (warp 0) =====
      // Address generation is hoisted out of the k-loop: per tile each thread precomputes, for its 8 rows, the
      // element offset of the filter-tap origin and a bit mask of the taps that fall inside the image; per k-block
      // only a (warp-uniform) tap offset is added.  wgrad rows change every k-block, so there each lane resolves ONE
      // pixel and the quarter-warps fetch it with shuffles.
      const int j = lane & 7;          // 16-byte column served by this thread
      const int q = lane >> 3;         // row within a group of 4
      uint32_t rs = 0, rph = 0;        // ring position: stage, phase (no division / modulo in the k-loop)
      for (int t = tile_first; t < tile_end; t += tile_step) {
        int split, m_tile, n_tile, kb_begin, nk;
        decode_tile(t, split, m_tile, n_tile, kb_begin, nk);
        const int n0 = n_tile * BN;
        long long off8[8];             // fprop/dgrad: origin offsets (elements) of the 8 rows this thread serves
        uint32_t mask8[8];             //              valid-tap bit masks
        int chunk_r = 0, chunk_s = 0, chunk_c0 = 0;
        bool chunk_ok = true;
        uint32_t tile_off = 0;
        if constexpr (!WGRAD) {
          // lane l resolves row l of this warp's 32 rows (one pixel decode per lane, not per served row) ...
          const RowPre rp = row_pre(P, pack_pixel(static_cast<long long>(m_tile) * BM + warp * 32 + lane, P));
          const bool rvalid = rp.yb > -(1 << 27);
          int oy = rp.yb, ox = rp.xb;
          if (P.transposed && P.stride == 2) { oy >>= 1; ox >>= 1; }
          const long long my_off = (static_cast<long long>(rp.nb + oy) * P.ws + ox) * P.cs;
          // per-axis tap validity (bit r of vy: filter row r lands inside the image; likewise vx for columns)
          uint32_t vy = 0, vx = 0;
          if (rvalid) {
            const int nky = P.kh, nkx = STEM ? 4 : P.kw;
            for (int r = 0; r < nky; ++r) {
              int h = P.transposed ? rp.yb - r : rp.yb + r;
              bool ok = true;
              if (P.transposed && P.stride == 2) { ok = (h & 1) == 0; h >>= 1; }
              vy |= (ok && static_cast<unsigned>(h) < static_cast<unsigned>(P.hs) ? 1u : 0u) << r;
            }
            for (int c = 0; c < nkx; ++c) {
              int w = P.transposed ? rp.xb - c : rp.xb + c;
              bool ok = true;
              if (P.transposed && P.stride == 2) { ok = (w & 1) == 0; w >>= 1; }
              vx |= (ok && static_cast<unsigned>(w) < static_cast<unsigned>(P.ws) ? 1u : 0u) << c;
            }
          }
          uint32_t my_mask;
          if constexpr (STEM) {
            my_mask = vy | (vx << 8);                     // taps r' in bits 0-3, column validity per s' in bits 8-11
          } else {
            my_mask = 0;
            for (int r = 0; r < P.kh; ++r)
              if ((vy >> r) & 1u) my_mask |= vx << (r * P.kw);
          }
          // ... and every thread fetches the 8 rows it serves
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int row = 4 * i + q;
            const long long o = __shfl_sync(0xffffffffu, my_off, row);
            const uint32_t m = __shfl_sync(0xffffffffu, my_mask, row);
            if constexpr (STEM) {
              off8[i] = o + (j >> 1) * P.cs + (j & 1) * 8;
              mask8[i] = ((m >> (8 + (j >> 1))) & 1u) ? (m & 0xFu) : 0u;
            } else {
              off8[i] = o + j * 8;
              mask8[i] = m;
            }
          }
          tile_off = warp * 32 * 128;
        } else {
          // warp = (chunk, half): 64 gathered channels x 32 of the 64 pixel rows of the k-block
          const int chunk = warp >> 1;
          const int gchunk = m_tile * 2 + chunk;           // 64-row chunk of the [K_total, Cout] result
          chunk_ok = gchunk < P.total_chunks;
          if constexpr (STEM) {
            chunk_r = gchunk;                              // filter row r'
          } else {
            uint32_t tap, cb, cr, csx;
            P.fd_cpb.divmod(static_cast<uint32_t>(gchunk), tap, cb);
            P.fd_kw.divmod(tap, cr, csx);
            chunk_c0 = static_cast<int>(cb) * 64;
            chunk_r = static_cast<int>(cr);
            chunk_s = static_cast<int>(csx);
          }
          tile_off = chunk * 8192 + (warp & 1) * 32 * 128;
        }
        int tc = 0, cb = 0;            // fprop/dgrad: visited-tap index and 64-channel block of the current k-block
        long long stem_toff = 0;
        for (int it = 0; it < nk; ++it) {
          const int s = static_cast<int>(rs);
          mbar_wait(empty_bar(s), rph ^ 1u);
          if (++rs == nstages) { rs = 0; rph ^= 1u; }
          const int kb = kb_begin + it;
          const uint32_t dst_base = a_addr(s) + tile_off;
          int kcoord = kb;             // fprop/dgrad: k-block of the weight matrix
          if constexpr (!WGRAD) {
            // warp-uniform tap offset (table filled on the host; counters instead of kb / cpb, tp / kw)
            int tp;
            long long toff;
            if constexpr (STEM) {
              tp = kb;
              toff = stem_toff;
              stem_toff += static_cast<long long>(P.ws) * P.cs;
            } else {
              tp = P.tap_list[tc];
              toff = P.tap_eoff[tc] + cb * 64;
              kcoord = tp * P.cpb + cb;
              if (++cb == P.cpb) { cb = 0; ++tc; }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int row = 4 * i + q;                   // row within this warp's 32 rows
              const bool ok = (mask8[i] >> tp) & 1u;
              const __nv_bfloat16* src = ok ? P.src + (off8[i] + toff) : P.src;
              cp_async16(dst_base + row * 128 + ((j ^ (row & 7)) << 4), src, ok ? 16u : 0u);
            }
          } else {
            // each lane resolves one of the warp's 32 pixels for this thread's fixed tap ...
            const uint32_t mypk = chunk_ok ? pack_pixel(static_cast<long long>(kb) * 64 + (warp & 1) * 32 + lane, P) : 0u;
            const RowPre rp = row_pre(P, mypk);
            bool myok;
            const __nv_bfloat16* myptr = tap_source(P, rp, chunk_r, STEM ? 0 : chunk_s, STEM ? 0 : chunk_c0, myok);
            const unsigned long long myaddr = reinterpret_cast<unsigned long long>(myptr);
            uint32_t okbits;                               // stem: validity per tap s' (4 bits); else 1 bit
            if constexpr (STEM) {
              okbits = 0;
              const bool rowok = (mypk >> 31) && static_cast<unsigned>(rp.yb + chunk_r) < static_cast<unsigned>(P.hs);
              for (int sp = 0; sp < 4; ++sp)
                okbits |= (rowok && static_cast<unsigned>(rp.xb + sp) < static_cast<unsigned>(P.ws) ? 1u : 0u) << sp;
            } else {
              okbits = myok ? 1u : 0u;
            }
            unsigned long long rowaddr = myaddr;
            if constexpr (STEM)   // origin of the filter row (tap s' = 0), may lie outside the image: used only when valid
              rowaddr = reinterpret_cast<unsigned long long>(
                  P.src + ((static_cast<long long>(rp.nb + rp.yb + chunk_r) * P.ws + rp.xb) * P.cs));
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int row = 4 * i + q;                   // ... and the quarter-warp serving that row fetches it
              const unsigned long long a = __shfl_sync(0xffffffffu, rowaddr, row);
              const uint32_t okb = __shfl_sync(0xffffffffu, okbits, row);
              const bool ok = STEM ? ((okb >> (j >> 1)) & 1u) : (okb & 1u);
              const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(a) + j * 8;   // stem: 4 taps x 16 channels are contiguous
              cp_async16(dst_base + row * 128 + ((j ^ (row & 7)) << 4), ok ? src : P.src, ok ? 16u : 0u);
            }
          }
          if (warp == 0) {
            if (elect_one()) {
              mbar_arrive_expect_tx(full_bar(s), C::kBBytes);
              if constexpr (!WGRAD) {
                tma_load_2d(b_addr(s), &tmap_b, full_bar(s), kcoord * BK, n0);
              } else {
#pragma unroll
                for (int i = 0; i < BN / 64; ++i)
                  tma_load_2d(b_addr(s) + i * 8192, &tmap_b, full_bar(s), n0 + 64 * i, kb * 64);
              }
            }
            __syncwarp();
          }
          // the mbarrier receives this thread's arrival when all of its cp.async above have landed (no wait here:
          // the ring depth alone bounds the loads in flight)
          cp_async_mbar_arrive_noinc(full_bar(s));
        }
      }
    } else if (warp == 0) {
      // ===== A and B by TMA (warp 0) =====
      // the whole warp walks the ring (converged); one elected lane issues.  Ring position and the (tap, channel
      // block) of the k-block are counters; tap coordinates come from the host-filled tables -- no division here.
      uint32_t rs = 0, rph = 0;
      for (int t = tile_first; t < tile_end; t += tile_step) {
        int split, m_tile, n_tile, kb_begin, nk;
        decode_tile(t, split, m_tile, n_tile, kb_begin, nk);
        const int n0 = n_tile * BN;
        int tile_w0 = 0, tile_h0 = 0, tile_n0 = 0;     // im2col base pixel of the tile's first GEMM row
        if constexpr (!WGRAD) {
          if (P.a_mode == 2) {
            uint32_t tn, rem, y0, x0;
            P.fd_hw.divmod(static_cast<uint32_t>(m_tile) * BM, tn, rem);
            P.fd_wm.divmod(rem, y0, x0);
            tile_n0 = static_cast<int>(tn);
            tile_w0 = static_cast<int>(x0) * P.i2c_stride + P.i2c_lo;
            tile_h0 = static_cast<int>(y0) * P.i2c_stride + P.i2c_lo;
          }
        }
        int tc = 0, cb = 0;                            // fprop/dgrad: visited-tap index, 64-channel block
        for (int it = 0; it < nk; ++it) {
          const int s = static_cast<int>(rs);
          mbar_wait(empty_bar(s), rph ^ 1u);
          if (++rs == nstages) { rs = 0; rph ^= 1u; }
          const int kb = kb_begin + it;
          if (elect_one()) {
            if constexpr (!WGRAD) {
              // A tile: 128 pixel rows x 64 channels (rows past the end / padding: zeros)
              mbar_arrive_expect_tx(full_bar(s), C::kBBytes + C::kABytes);
              if (P.a_mode == 1)
                tma_load_2d(a_addr(s), &tmap_a, full_bar(s), kb * BK, m_tile * BM);
              else   // dgrad: dy pixel (y + pad - r, x + pad - s) = base + (k-1-r, k-1-s): flipped in the table
                tma_load_im2col_4d(a_addr(s), &tmap_a, full_bar(s), cb * BK, tile_w0, tile_h0, tile_n0,
                                   P.tap_s[tc], P.tap_r[tc]);
              tma_load_2d(b_addr(s), &tmap_b, full_bar(s), (P.tap_list[tc] * P.cpb + cb) * BK, n0);
            } else {
              // A tile: 64 pixels x (up to) two 64-channel chunks, MN-major like the dY tile
              const int nchunks = min(2, P.total_chunks - 2 * m_tile);
              mbar_arrive_expect_tx(full_bar(s), C::kBBytes + nchunks * 8192);
              if (P.a_mode == 1) {
                for (int i = 0; i < nchunks; ++i)
                  tma_load_2d(a_addr(s) + i * 8192, &tmap_a, full_bar(s), (2 * m_tile + i) * 64, kb * 64);
              } else {
                // the k-block's first pixel -> base pixel; every chunk = (filter tap, 64 channels)
                uint32_t n0i, rem, y0, x0;
                P.fd_hw.divmod(static_cast<uint32_t>(kb) * 64u, n0i, rem);
                P.fd_wm.divmod(rem, y0, x0);
                for (int i = 0; i < nchunks; ++i) {
                  uint32_t tap, cbk, r, sx;
                  P.fd_cpb.divmod(static_cast<uint32_t>(2 * m_tile + i), tap, cbk);
                  P.fd_kw.divmod(tap, r, sx);
                  tma_load_im2col_4d(a_addr(s) + i * 8192, &tmap_a, full_bar(s), static_cast<int>(cbk) * 64,
                                     static_cast<int>(x0) * P.i2c_stride + P.i2c_lo,
                                     static_cast<int>(y0) * P.i2c_stride + P.i2c_lo, static_cast<int>(n0i),
                                     static_cast<uint16_t>(sx), static_cast<uint16_t>(r));
                }
              }
#pragma unroll
              for (int i = 0; i < BN / 64; ++i)
                tma_load_2d(b_addr(s) + i * 8192, &tmap_b, full_bar(s), n0 + 64 * i, kb * 64);
            }
          }
          if constexpr (!WGRAD) {
            if (++cb == P.cpb) { cb = 0; ++tc; }
          }
          __syncwarp();
        }
      }
    }
    return;    // producers are done; the consumers below synchronise among themselves only
  }

  // ===== consumers (warpgroups 1, 2) =====
  const int g = (warp >> 2) - 1;                  // tile rows [64 g, 64 g + 64)
  const int wq = warp & 3;                        // fragment rows [16 wq, 16 wq + 16) of the warpgroup's 64
  const int ew = g * 4 + wq;                      // consumer warp 0..7: staging tile / statistics slot
  const int fr = lane >> 2, fc = 2 * (lane & 3);  // fragment row / first column of this lane
  float* const stat_sm = reinterpret_cast<float*>(smem_gen + C::kStatOffset) + ew * (2 * BN);
  if constexpr (!WGRAD) {
    if (P.stat_out != nullptr)
      for (int i = lane; i < 2 * BN; i += 32) stat_sm[i] = 0.f;
  }
  // K-major: 8-row atoms 1024 B apart; MN-major: 64-wide chunks 8192 B apart (LBO), 8-k atoms 1024 B (SBO).  This
  // warpgroup's 64 A rows (wgrad: its 64-channel chunk) start 8192 B into the stage.
  constexpr uint32_t kLbo = WGRAD ? 8192u : 16u;
  constexpr uint32_t kadv = WGRAD ? (2048u >> 4) : (32u >> 4);   // one k16 step, in 16-byte units
  constexpr int kT = WGRAD ? 1 : 0;
  float acc[BN / 2];
  uint32_t rs = 0, rph = 0;
  for (int t = tile_first; t < tile_end; t += tile_step) {
    int split, m_tile, n_tile, kb_begin, nk;
    decode_tile(t, split, m_tile, n_tile, kb_begin, nk);
    int prev = 0;
    for (int it = 0; it < nk; ++it) {
      const int s = static_cast<int>(rs);
      mbar_wait(full_bar(s), rph);
      if (++rs == nstages) { rs = 0; rph ^= 1u; }
      if constexpr (!ATMA) fence_proxy_async();   // the gathered rows were written through the generic proxy
      const uint64_t adesc = make_smem_desc(a_addr(s) + g * 8192, kLbo, 1024u);
      const uint64_t bdesc = make_smem_desc(b_addr(s), kLbo, 1024u);
      wgmma_fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        wgmma_bf16<BN, kT, kT>(acc, adesc + static_cast<uint64_t>(k * kadv), bdesc + static_cast<uint64_t>(k * kadv),
                               (it > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_fence_operands(acc);
      // one k-block stays in flight: once the previous one has completed, its stage goes back to the producer
      if (it > 0) {
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (nk > 0 && lane == 0) mbar_arrive(empty_bar(prev));
    const int n0 = n_tile * BN;

    if constexpr (!WGRAD) {
      // registers -> bf16 staging tile -> coalesced row stores; BN statistics / moments sum the staged (stored) values
      const uint32_t stage_base = smem_base + C::kEpiOffset + ew * C::kEpiWarpBytes;
      const bool relu_now = AFFINE && P.epi_relu && P.epi_res == nullptr;    // with a residual the ReLU follows the add
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + fc;
        float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
        if constexpr (AFFINE) {
          const float2 a = __ldg(reinterpret_cast<const float2*>(P.epi_scale + n0 + col));
          const float2 b = __ldg(reinterpret_cast<const float2*>(P.epi_shift + n0 + col));
          v0 = fmaf(v0, a.x, b.x); v1 = fmaf(v1, a.y, b.y); v2 = fmaf(v2, a.x, b.x); v3 = fmaf(v3, a.y, b.y);
          if (relu_now) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
        }
        __nv_bfloat162 h0 = __floats2bfloat162_rn(v0, v1), h1 = __floats2bfloat162_rn(v2, v3);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(stage_base + fr * C::kStageRowBytes + col * 2),
                     "r"(*reinterpret_cast<uint32_t*>(&h0)) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(stage_base + (fr + 8) * C::kStageRowBytes + col * 2),
                     "r"(*reinterpret_cast<uint32_t*>(&h1)) : "memory");
      }
      __syncwarp();
      constexpr int kLanesPerRow = BN * 2 / 16;           // 16-byte pieces of one output row
      constexpr int kRowsPerIter = 32 / kLanesPerRow;
      constexpr int kIters = 16 / kRowsPerIter;
      const int sub = lane / kLanesPerRow, col16 = lane % kLanesPerRow;
      const long long p0 = static_cast<long long>(m_tile) * BM + g * 64 + wq * 16;
      __nv_bfloat16* out_cols = reinterpret_cast<__nv_bfloat16*>(P.out) + n0 + col16 * 8;
#pragma unroll
      for (int i = 0; i < kIters; ++i) {
        const int rl = i * kRowsPerIter + sub;
        const long long p = p0 + rl;
        // output row (32-bit: the host checks that the output has fewer than 2^31 rows)
        int orow = (p < P.pixels && nk > 0) ? static_cast<int>(p) : -1;
        if (orow >= 0 && P.cls_on) {                          // class pixel -> row of the full image
          const uint32_t pk = pack_pixel(p, P);
          const int n = (pk >> 18) & 0x1FFF, yy = (pk >> 9) & 0x1FF, xx = pk & 0x1FF;
          orow = (n * P.full_h + 2 * yy + P.cls_py) * P.full_w + 2 * xx + P.cls_px;
        }
        if (orow >= 0) {
          uint4 val;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(val.x), "=r"(val.y), "=r"(val.z), "=r"(val.w)
                       : "r"(stage_base + rl * C::kStageRowBytes + col16 * 16));
          if constexpr (AFFINE) {
            if (P.epi_res != nullptr) {
              const uint4 rv = *reinterpret_cast<const uint4*>(P.epi_res + n0 + col16 * 8 + static_cast<long long>(orow) * P.ldc);
              uint32_t o[4] = {val.x, val.y, val.z, val.w};
              const uint32_t rr[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                float lo = __uint_as_float(o[e] << 16) + __uint_as_float(rr[e] << 16);
                float hi = __uint_as_float(o[e] & 0xffff0000u) + __uint_as_float(rr[e] & 0xffff0000u);
                if (P.epi_relu) { lo = fmaxf(lo, 0.f); hi = fmaxf(hi, 0.f); }
                __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
                o[e] = *reinterpret_cast<uint32_t*>(&h);
              }
              val = make_uint4(o[0], o[1], o[2], o[3]);
            }
          }
          *reinterpret_cast<uint4*>(out_cols + static_cast<long long>(orow) * P.ldc) = val;
        }
      }
      if (BSTAT || P.stat_out != nullptr) {
        // lane l owns the column pairs l (and l + 32 at BN = 128) of the tile: one bf16x2 word per staged row (rows
        // past the end of the tensor hold zeros: their A rows were zero-filled)
#pragma unroll
        for (int h = 0; h < BN / 64; ++h) {
          const int col = 2 * (lane + 32 * h);
          float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
          float2 bsc = make_float2(0.f, 0.f), bsh = bsc;
          if constexpr (BSTAT) {
            bsc = __ldg(reinterpret_cast<const float2*>(P.bst_scale + n0 + col));
            bsh = __ldg(reinterpret_cast<const float2*>(P.bst_shift + n0 + col));
          }
#pragma unroll
          for (int r = 0; r < 16; ++r) {
            uint32_t w;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(stage_base + r * C::kStageRowBytes + col * 2));
            float g0 = __uint_as_float(w << 16), g1 = __uint_as_float(w & 0xffff0000u);
            if constexpr (BSTAT) {
              // dz = g * [bn(y) > 0] with the forward's own fmaf; S0 += dz, S1 += dz * y
              const long long p = p0 + r;
              const uint32_t yw = p < P.pixels ? __ldg(reinterpret_cast<const unsigned int*>(P.bst_y + p * P.ldc + n0 + col)) : 0u;
              const float y0 = __uint_as_float(yw << 16), y1 = __uint_as_float(yw & 0xffff0000u);
              if (!(fmaf(y0, bsc.x, bsh.x) > 0.f)) g0 = 0.f;
              if (!(fmaf(y1, bsc.y, bsh.y) > 0.f)) g1 = 0.f;
              s0 += g0; s1 += g1;
              q0 = fmaf(g0, y0, q0); q1 = fmaf(g1, y1, q1);
            } else {
              s0 += g0; s1 += g1;
              q0 = fmaf(g0, g0, q0); q1 = fmaf(g1, g1, q1);
            }
          }
          stat_sm[col] += s0;
          stat_sm[col + 1] += s1;
          stat_sm[BN + col] += q0;
          stat_sm[BN + col + 1] += q1;
        }
      }
      __syncwarp();                                         // staging tile is reused by the next tile
    } else {
      // partials are stored TRANSPOSED, [split][Cout][K_total] (the reduce kernel walks k)
      const int ktot = P.total_chunks * 64;
      const int krow = m_tile * BM + g * 64 + wq * 16 + fr;   // row of the [K_total, Cout] result
      float* out = reinterpret_cast<float*>(P.out) + (static_cast<size_t>(split) * P.ldc + n0) * ktot;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const size_t c0 = static_cast<size_t>(8 * j + fc) * ktot;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (krow < ktot) out[c0 + e * ktot + krow] = nk > 0 ? acc[4 * j + e] : 0.f;
          if (krow + 8 < ktot) out[c0 + e * ktot + krow + 8] = nk > 0 ? acc[4 * j + 2 + e] : 0.f;
        }
      }
    }
  }
  if constexpr (!WGRAD) {
    if (P.stat_out != nullptr) {
      // one flush per CTA: the eight consumer warps' smem column sums are combined (fixed order -> deterministic) and
      // written as stat_out[blockIdx.x][0][c] = sums, [1][c] = sums of squares for the BN columns of this CTA's
      // n_tile.  Every CTA of the launch owns >= 1 tile (grid <= tiles), so every row of its n_tile's column range
      // is written: the consumer (bn_finalize) reads exactly those, no zero-fill needed.
      asm volatile("bar.sync 1, 256;" ::: "memory");       // the two consumer warpgroups
      const float* all = reinterpret_cast<const float*>(smem_gen + C::kStatOffset);
      float* dst = P.stat_out + static_cast<size_t>(blockIdx.x) * 2 * P.ldc + fixed_n * BN;
      for (int o = static_cast<int>(threadIdx.x) - kProducerThreads; o < 2 * BN; o += kThreads - kProducerThreads) {
        const int k = o / BN, col = o - k * BN;
        const float v = ((all[o] + all[2 * BN + o]) + (all[4 * BN + o] + all[6 * BN + o])) +
                        ((all[8 * BN + o] + all[10 * BN + o]) + (all[12 * BN + o] + all[14 * BN + o]));
        dst[static_cast<size_t>(k) * P.ldc + col] = v;
      }
    }
  }
}

// --------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 tensor [outer][inner] (inner contiguous), box = 64 x box_outer, 128-byte swizzle.
int make_tmap_bf16_2d(CUtensorMap* tm, const void* ptr, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                      uint32_t box_outer) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return DIRB200_ERR_CUDA;
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {64, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) inner=%llu outer=%llu stride=%llu", (int)r,
              (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)row_stride_bytes);
    return DIRB200_ERR_CUDA;
  }
  return DIRB200_OK;
}

// im2col-mode map of an NHWC bf16 tensor: 64 channels x `pixels_per_col` output positions per load, 128-byte swizzle.
// lower / upper: offsets of the base-pixel bounding box from 0 / from the extent (same for W and H); trav: traversal
// stride (= conv stride).  Parameters as cutlass/conv/collective/detail.hpp derives them (fprop: lower = -pad,
// upper = pad - (k - 1); dgrad: lower = pad - (k - 1), upper = lower + extent(dx) - extent(dy)).
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
int make_tmap_im2col_bf16(CUtensorMap* tm, const void* ptr, int c, int w, int h, int n, int lower_w, int lower_h,
                          int upper_w, int upper_h, int trav, int pixels_per_col) {
  static EncodeIm2colFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeIm2colFn>(p);
  }
  if (!fn) {
    set_error("cuTensorMapEncodeIm2col entry point not available");
    return DIRB200_ERR_CUDA;
  }
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)c * 2, (cuuint64_t)w * c * 2, (cuuint64_t)h * w * c * 2};
  int lower[2] = {lower_w, lower_h}, upper[2] = {upper_w, upper_h};
  cuuint32_t estr[4] = {1, (cuuint32_t)trav, (cuuint32_t)trav, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower, upper, 64,
                  (cuuint32_t)pixels_per_col, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (%d) c=%d w=%d h=%d n=%d lower=%d,%d upper=%d,%d stride=%d", (int)r, c, w, h,
              n, lower_w, lower_h, upper_w, upper_h, trav);
    return DIRB200_ERR_CUDA;
  }
  // same driver workaround as cute's make_im2col_tma_copy_desc (drivers <= 13.1, tensors < 128 KiB)
  int drv = 0;
  if (cudaDriverGetVersion(&drv) == cudaSuccess && drv <= 13010 && (size_t)c * w * h * n * 2 < 131072)
    reinterpret_cast<uint64_t*>(tm)[1] &= ~(1ull << 21);
  return DIRB200_OK;
}

// Host-side completion of the launch parameters: reciprocal constants for every run-time divisor the kernel meets and
// the per-tap tables (gather offset, im2col offsets) indexed by the position in tap_list.
static IgemmParams finish_params(const IgemmParams& P) {
  IgemmParams Q = P;
  Q.fd_hw = make_fastdiv(static_cast<uint32_t>(Q.hm * Q.wm));
  Q.fd_wm = make_fastdiv(static_cast<uint32_t>(Q.wm));
  Q.fd_cpb = make_fastdiv(static_cast<uint32_t>(Q.cpb > 0 ? Q.cpb : 1));
  Q.fd_kw = make_fastdiv(static_cast<uint32_t>(Q.kw > 0 ? Q.kw : 1));
  Q.fd_ntiles = make_fastdiv(static_cast<uint32_t>(Q.n_tiles > 0 ? Q.n_tiles : 1));
  Q.fd_persplit = make_fastdiv(static_cast<uint32_t>(Q.m_tiles * Q.n_tiles > 0 ? Q.m_tiles * Q.n_tiles : 1));
  const int nt = Q.ntaps_c < kMaxTaps ? Q.ntaps_c : kMaxTaps;
  for (int i = 0; i < kMaxTaps; ++i) {
    Q.tap_eoff[i] = 0;
    Q.tap_r[i] = Q.tap_s[i] = 0;
  }
  for (int i = 0; i < nt && Q.kw > 0; ++i) {
    const int tp = Q.tap_list[i];
    int r = tp / Q.kw, sx = tp - r * Q.kw;
    if (Q.transposed && Q.cls_on) {
      // parity class of a stride-2 dgrad: tap (r, s) reads dy pixel (y' + (py + pad - r) / 2, x' + (px + pad - s) / 2);
      // im2col offsets are relative to the base-pixel box's lower corner i2c_lo
      Q.tap_r[i] = static_cast<unsigned short>((Q.cls_py + Q.pad - r) / 2 - Q.i2c_lo);
      Q.tap_s[i] = static_cast<unsigned short>((Q.cls_px + Q.pad - sx) / 2 - Q.i2c_lo);
      r >>= 1; sx >>= 1;
      Q.tap_eoff[i] = -static_cast<long long>(r * Q.ws + sx) * Q.cs;
    } else if (Q.transposed) {
      Q.tap_r[i] = static_cast<unsigned short>(Q.kh - 1 - r);
      Q.tap_s[i] = static_cast<unsigned short>(Q.kw - 1 - sx);
      if (Q.stride == 2) { r >>= 1; sx >>= 1; }
      Q.tap_eoff[i] = -static_cast<long long>(r * Q.ws + sx) * Q.cs;
    } else {
      Q.tap_r[i] = static_cast<unsigned short>(r);
      Q.tap_s[i] = static_cast<unsigned short>(sx);
      Q.tap_eoff[i] = static_cast<long long>(r * Q.ws + sx) * Q.cs;
    }
  }
  return Q;
}

template <int BN, bool WGRAD, bool STEM, bool ATMA = false, bool AFFINE = false, bool BSTAT = false>
static int launch_igemm_impl(const CUtensorMap& tm, const CUtensorMap& tma, const IgemmParams& Qin, int grid,
                             cudaStream_t st) {
  using C = Cfg<BN, !WGRAD>;
  const IgemmParams Q = finish_params(Qin);
  static bool configured = false;
  if (!configured) {
    DIRB_CUDA(cudaFuncSetAttribute(igemm_kernel<BN, WGRAD, STEM, ATMA, AFFINE, BSTAT>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes));
    configured = true;
  }
  igemm_kernel<BN, WGRAD, STEM, ATMA, AFFINE, BSTAT><<<grid, kThreads, C::kSmemBytes, st>>>(tm, tma, Q);
  DIRB_LAUNCHED();
  return DIRB200_OK;
}

// tma != nullptr: the A operand is loaded by TMA too (tiled or im2col map, P.a_mode)
template <int BN, bool WGRAD, bool STEM>
static int launch_igemm(const CUtensorMap& tm, const IgemmParams& Q, int grid, cudaStream_t st,
                        const CUtensorMap* tma = nullptr) {
  if constexpr (!STEM) {
    if (tma) {
      if constexpr (!WGRAD) {
        if (Q.epi_scale != nullptr) return launch_igemm_impl<BN, false, false, true, true>(tm, *tma, Q, grid, st);
        if (Q.bst_y != nullptr) return launch_igemm_impl<BN, false, false, true, false, true>(tm, *tma, Q, grid, st);
      }
      return launch_igemm_impl<BN, WGRAD, false, true>(tm, *tma, Q, grid, st);
    }
  }
  if constexpr (!WGRAD && !STEM) {
    // gather-fed fprop (DIRB200_ATMA=0 / DIRB200_IM2COL=0): the folded-BN epilogue works the same way
    if (Q.epi_scale != nullptr) return launch_igemm_impl<BN, false, false, false, true>(tm, tm, Q, grid, st);
  }
  if (Q.epi_scale != nullptr || Q.bst_y != nullptr) {
    set_error("conv: the BN-backward moments epilogue needs a TMA-fed A operand; the folded-BN one a non-stem fprop");
    return DIRB200_ERR_ARG;
  }
  return launch_igemm_impl<BN, WGRAD, STEM>(tm, tm, Q, grid, st);
}

// GEMM-N tile width: 128 where N allows (a consumer warpgroup's 64 x 128 fp32 accumulators take 64 registers per
// thread; a 256-wide tile would need 128 and leave too few for the epilogue at three warpgroups per SM), else 64.
static int pick_bn(int n_dim) { return n_dim % 128 == 0 ? 128 : 64; }

#define DISPATCH_BN(bn, WG, ST, ...) \
  ((bn) == 128 ? launch_igemm<128, WG, ST>(__VA_ARGS__) : launch_igemm<64, WG, ST>(__VA_ARGS__))

static int check_shape(const ConvShape& s, bool stem, const char* who) {
  DIRB_CHECK_ARG(s.n > 0 && s.h > 0 && s.w > 0 && s.kh > 0 && s.kw > 0 && s.stride > 0 && s.pad >= 0,
                 "%s: bad conv shape", who);
  DIRB_CHECK_ARG(s.cout % 64 == 0, "%s: Cout must be a multiple of 64 (got %d)", who, s.cout);
  DIRB_CHECK_ARG(static_cast<long long>(s.n) * s.h * s.w < (1LL << 31) && static_cast<long long>(s.n) * s.ho * s.wo < (1LL << 31),
                 "%s: more than 2^31 pixels", who);
  if (stem)
    DIRB_CHECK_ARG(s.cin == 16 && s.kh == 4 && s.kw == 4 && s.stride == 1, "%s: stem expects the 4x4x16 s2d form", who);
  else
    DIRB_CHECK_ARG(s.cin % 64 == 0, "%s: Cin must be a multiple of 64 (got %d)", who, s.cin);
  return DIRB200_OK;
}

// DIRB200_ATMA=0 keeps the cp.async gather for every layer (A/B measurements); default: 1x1 stride-1 GEMMs take the
// A operand through TMA.
static bool atma_enabled() {
  static const bool on = env_switch("DIRB200_ATMA");
  return on;
}
// DIRB200_IM2COL=0: the cp.async gather for the convs that would take im2col-mode TMA.
static bool im2col_enabled() {
  static const bool on = env_switch("DIRB200_IM2COL");
  return on && atma_enabled();
}

// Split-K factor of the wgrad GEMM (K = pixels).  The persistent CTAs walk tiles x splits work items in waves of
// num_sms; one item costs its k-blocks plus an epilogue worth ~6 k-blocks (128 x BN fp32 partials; an estimate, not
// re-measured on H100), so a launch costs about waves x (k-blocks per split + 6); the minimiser avoids straggler waves.
static int wgrad_splits(int kblocks, int tiles) {
  const int sms = num_sms();
  int max_splits = (kblocks + 7) / 8;                   // at least 8 k-blocks per split
  if (max_splits < 1) max_splits = 1;
  int hi = (4 * sms + tiles - 1) / tiles;
  if (hi > max_splits) hi = max_splits;
  int best = 1;
  long long best_cost = -1;
  for (int sp = 1; sp <= hi; ++sp) {
    const long long waves = (static_cast<long long>(tiles) * sp + sms - 1) / sms;
    const long long per = (kblocks + sp - 1) / sp;
    const long long cost = waves * (per + 6);
    if (best_cost < 0 || cost < best_cost) {
      best_cost = cost;
      best = sp;
    }
  }
  return best;
}

int plan_conv(const ConvShape& s, bool stem, int op, ConvPlan* pl) {
  static const char* const kWho[3] = {"conv_fprop", "conv_dgrad", "conv_wgrad"};
  *pl = ConvPlan{};
  if (int rc = check_shape(s, stem, kWho[op])) return rc;
  const bool dgrad = op == 1, wgrad = op == 2;
  const int taps = s.kh * s.kw;
  DIRB_CHECK_ARG(!(dgrad && stem), "conv_dgrad: the stem has no data gradient");
  DIRB_CHECK_ARG(!dgrad || s.stride == 1 || s.stride == 2, "conv_dgrad: stride must be 1 or 2 (got %d)", s.stride);
  const int max_taps = dgrad && s.stride == 2 ? 9 : kMaxTaps;
  DIRB_CHECK_ARG(stem || taps <= max_taps, "%s: at most %d filter taps (got %dx%d)", kWho[op], max_taps, s.kh, s.kw);

  pl->op = op;
  pl->stem = stem;
  const int n_dim = dgrad ? s.cin : s.cout;
  const int cs = dgrad ? s.cout : s.cin;        // channels of the gathered tensor (dgrad: dy)
  pl->bn = pick_bn(n_dim);
  pl->n_tiles = n_dim / pl->bn;
  // A operand: 1x1 stride-1 GEMMs read a plain [pixels][channels] matrix by tiled TMA; every other non-stem conv takes
  // im2col-mode TMA, except a stride-1 dgrad with a non-square filter (one box offset serves both axes there); the stem
  // keeps the cp.async gather
  const bool plain = !stem && s.kh == 1 && s.kw == 1 && s.stride == 1 && s.pad == 0 && atma_enabled();
  pl->a_form = plain ? 1 : (!stem && im2col_enabled() && !(dgrad && s.stride == 1 && s.kh != s.kw)) ? 2 : 0;
  pl->fuses_bn_moments = dgrad && s.stride == 1 && pl->a_form != 0;
  pl->classes = dgrad && s.stride == 2;
  pl->splits = 1;

  for (int cls = 0; cls < (pl->classes ? 4 : 1); ++cls) {
    ConvLaunch L{};
    if (pl->classes) {
      // output pixels (2y' + py, 2x' + px) receive only the taps whose parity matches: quarter-size grids
      L.cls_py = cls >> 1;
      L.cls_px = cls & 1;
      L.hm = (s.h - L.cls_py + 1) / 2;
      L.wm = (s.w - L.cls_px + 1) / 2;
      for (int r = 0; r < s.kh; ++r)
        for (int q = 0; q < s.kw; ++q)
          if (((L.cls_py + s.pad - r) & 1) == 0 && ((L.cls_px + s.pad - q) & 1) == 0) L.taps[L.ntaps++] = r * s.kw + q;
      if (L.ntaps == 0) pl->need_zero = true;
      if (L.ntaps == 0 || L.hm <= 0 || L.wm <= 0) continue;
      L.num_kblocks = L.ntaps * (cs / 64);
    } else {
      L.hm = dgrad ? s.h : s.ho;
      L.wm = dgrad ? s.w : s.wo;
      L.ntaps = taps;
      for (int i = 0; i < kMaxTaps; ++i) L.taps[i] = i;
      L.num_kblocks = taps * cs / 64;
    }
    L.pixels = static_cast<long long>(s.n) * L.hm * L.wm;
    if (wgrad) {
      L.num_kblocks = static_cast<int>((L.pixels + 63) / 64);
      L.m_tiles = (taps * cs / 64 + 1) / 2;         // pairs of 64-row chunks of the K_total x Cout result
      pl->splits = wgrad_splits(L.num_kblocks, L.m_tiles * pl->n_tiles);
      pl->kblocks_per_split = (L.num_kblocks + pl->splits - 1) / pl->splits;
      pl->workspace_bytes = static_cast<size_t>(pl->splits) * taps * s.cin * s.cout * sizeof(float);
    } else {
      L.m_tiles = static_cast<int>((L.pixels + BM - 1) / BM);
    }
    if (pl->a_form == 2 && !dgrad) {              // x [n,h,w,cin], base pixel (ho*stride - pad, wo*stride - pad)
      L.i2c_stride = s.stride;
      L.i2c_lo = L.i2c_lower_w = L.i2c_lower_h = -s.pad;
      L.i2c_upper_w = s.pad - (s.kw - 1);
      L.i2c_upper_h = s.pad - (s.kh - 1);
    } else if (pl->a_form == 2) {
      // dy [n,ho,wo,cout]: a stride-1 "convolution" over the dy grid whose taps sit at offsets pad - r (tap offsets
      // reversed) or, for a parity class, (py + pad - r) / 2; the base-pixel box is [lo, lo + row grid) with lo the
      // lowest offset (out-of-range dy pixels arrive as zeros)
      int lo = s.pad - (s.kh - 1);
      if (pl->classes) {
        lo = 1 << 20;
        for (int i = 0; i < L.ntaps; ++i) {
          const int r = L.taps[i] / s.kw, q = L.taps[i] % s.kw;
          const int orr = (L.cls_py + s.pad - r) / 2, oq = (L.cls_px + s.pad - q) / 2;
          lo = orr < lo ? orr : lo;
          lo = oq < lo ? oq : lo;
        }
      }
      L.i2c_stride = 1;
      L.i2c_lo = L.i2c_lower_w = L.i2c_lower_h = lo;
      L.i2c_upper_w = lo + L.wm - s.wo;
      L.i2c_upper_h = lo + L.hm - s.ho;
    }
    const int tiles = L.m_tiles * pl->n_tiles * pl->splits;
    L.grid = tiles < num_sms() ? tiles : num_sms();
    // fprop / dgrad CTAs each keep one n_tile: at least one CTA per n_tile, also when DIRB200_SMS caps the SM count
    // below the tile count (the extra CTAs run as a second wave)
    if (!wgrad && L.grid < pl->n_tiles) L.grid = pl->n_tiles;
    pl->launch[pl->nlaunch++] = L;
  }
  if (!wgrad && !pl->classes) pl->layout = StatLayout{pl->launch[0].grid, pl->n_tiles, pl->bn, 1};
  return DIRB200_OK;
}

// Runs every launch of a plan.  P0 holds the tensor pointers (src: the gathered tensor, out) and the epilogue
// options; b is the B operand (fprop / dgrad: the weights [N][K], K-major; wgrad: dy [pixels][cout]).
static int run_plan(const ConvShape& s, const ConvPlan& pl, const IgemmParams& P0, const void* b, cudaStream_t st) {
  const bool dgrad = pl.op == 1, wgrad = pl.op == 2;
  CUtensorMap tm;
  if (wgrad) {
    if (int rc = make_tmap_bf16_2d(&tm, b, s.cout, static_cast<uint64_t>(pl.launch[0].pixels),
                                   static_cast<uint64_t>(s.cout) * 2, 64))
      return rc;
  } else {
    const int ktot = s.kh * s.kw * (dgrad ? s.cout : s.cin);
    if (int rc = make_tmap_bf16_2d(&tm, b, ktot, dgrad ? s.cin : s.cout, static_cast<uint64_t>(ktot) * 2, pl.bn))
      return rc;
  }
  if (pl.need_zero)
    DIRB_CUDA(cudaMemsetAsync(P0.out, 0, static_cast<size_t>(s.n) * s.h * s.w * s.cin * sizeof(__nv_bfloat16), st));
  for (int i = 0; i < pl.nlaunch; ++i) {
    const ConvLaunch& L = pl.launch[i];
    IgemmParams P = P0;
    P.n = s.n;
    P.hs = dgrad ? s.ho : s.h;
    P.ws = dgrad ? s.wo : s.w;
    P.cs = dgrad ? s.cout : s.cin;
    P.hm = L.hm;
    P.wm = L.wm;
    P.kh = s.kh; P.kw = s.kw; P.stride = s.stride; P.pad = s.pad; P.transposed = dgrad ? 1 : 0;
    if (pl.classes) {
      P.cls_on = 1; P.cls_py = L.cls_py; P.cls_px = L.cls_px; P.full_h = s.h; P.full_w = s.w;
    }
    P.ntaps_c = L.ntaps;
    for (int t = 0; t < kMaxTaps; ++t) P.tap_list[t] = L.taps[t];
    P.cpb = pl.stem ? 1 : P.cs / 64;
    P.pixels = L.pixels;
    P.num_kblocks = L.num_kblocks;
    P.kblocks_per_split = pl.kblocks_per_split;
    if (wgrad) P.total_chunks = s.kh * s.kw * s.cin / 64;
    P.m_tiles = L.m_tiles;
    P.n_tiles = pl.n_tiles;
    P.num_tiles = L.m_tiles * pl.n_tiles * pl.splits;
    P.a_mode = pl.a_form;
    P.i2c_stride = L.i2c_stride;
    P.i2c_lo = L.i2c_lo;
    P.ldc = dgrad ? s.cin : s.cout;
    // the A operand's map: the gathered tensor as a plain [pixels][channels] matrix, or in im2col mode; boxes of
    // 64 channels x one tile's rows (wgrad: one 64-pixel k-block)
    const uint32_t rows = wgrad ? 64 : BM;
    CUtensorMap ta;
    if (pl.a_form == 1) {
      if (int rc = make_tmap_bf16_2d(&ta, P.src, P.cs, static_cast<uint64_t>(P.pixels), static_cast<uint64_t>(P.cs) * 2,
                                     rows))
        return rc;
    } else if (pl.a_form == 2) {
      if (int rc = make_tmap_im2col_bf16(&ta, P.src, P.cs, P.ws, P.hs, P.n, L.i2c_lower_w, L.i2c_lower_h, L.i2c_upper_w,
                                         L.i2c_upper_h, L.i2c_stride, rows))
        return rc;
    }
    const CUtensorMap* pa = pl.a_form != 0 ? &ta : nullptr;
    int rc;
    if (pl.stem)
      rc = wgrad ? DISPATCH_BN(pl.bn, true, true, tm, P, L.grid, st) : DISPATCH_BN(pl.bn, false, true, tm, P, L.grid, st);
    else
      rc = wgrad ? DISPATCH_BN(pl.bn, true, false, tm, P, L.grid, st, pa)
                 : DISPATCH_BN(pl.bn, false, false, tm, P, L.grid, st, pa);
    if (rc) return rc;
  }
  return DIRB200_OK;
}

// Y[n,ho,wo,cout] = conv(X[n,h,w,cin], W[cout][kh][kw][cin])
static int conv_fprop_impl(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* y, const ConvShape& s, bool stem,
                           cudaStream_t st, float* stat_partial, const ConvEpilogue* epi, StatLayout* layout) {
  ConvPlan pl;
  if (int rc = plan_conv(s, stem, 0, &pl)) return rc;
  IgemmParams P{};
  P.src = x; P.out = y;
  P.stat_out = stat_partial;
  if (epi) {
    P.epi_scale = epi->scale; P.epi_shift = epi->shift; P.epi_res = epi->residual; P.epi_relu = epi->relu ? 1 : 0;
  }
  if (int rc = run_plan(s, pl, P, w, st)) return rc;
  if (layout) *layout = pl.layout;
  return DIRB200_OK;
}

int conv_fprop(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* y, const ConvShape& s, bool stem,
               cudaStream_t st, float* stat_partial, StatLayout* layout) {
  return conv_fprop_impl(x, w, y, s, stem, st, stat_partial, nullptr, layout);
}

int conv_fprop_affine(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* out, const ConvShape& s,
                      const ConvEpilogue& epi, cudaStream_t st) {
  DIRB_CHECK_ARG(epi.scale && epi.shift, "conv_fprop_affine: scale / shift missing");
  return conv_fprop_impl(x, w, out, s, false, st, nullptr, &epi, nullptr);
}

// dX[n,h,w,cin] = conv_transpose(dY[n,ho,wo,cout], Wt[cin][kh][kw][cout]); stride 2: one launch per output-pixel
// parity class, a class without any tap receives no gradient (zeros)
int conv_dgrad(const __nv_bfloat16* dy, const __nv_bfloat16* wt, __nv_bfloat16* dx, const ConvShape& s,
               cudaStream_t st, const DgradBnMoments* bnm) {
  ConvPlan pl;
  if (int rc = plan_conv(s, false, 1, &pl)) return rc;
  DIRB_CHECK_ARG(!bnm || (pl.fuses_bn_moments && bnm->y && bnm->scale && bnm->shift && bnm->partial),
                 "conv_dgrad: BN-backward moments are fused into TMA-fed stride-1 dgrads only");
  IgemmParams P{};
  P.src = dy; P.out = dx;
  if (bnm) {
    P.bst_y = bnm->y; P.bst_scale = bnm->scale; P.bst_shift = bnm->shift; P.stat_out = bnm->partial;
  }
  if (int rc = run_plan(s, pl, P, wt, st)) return rc;
  if (bnm && bnm->layout) *bnm->layout = pl.layout;
  return DIRB200_OK;
}

// partial[split][cout][(r,s,c)] = sum over the split's pixels of X_gathered^T dY
int conv_wgrad_partials(const __nv_bfloat16* x, const __nv_bfloat16* dy, float* partial, const ConvShape& s, bool stem,
                        int* splits_out, cudaStream_t st) {
  ConvPlan pl;
  if (int rc = plan_conv(s, stem, 2, &pl)) return rc;
  IgemmParams P{};
  P.src = x; P.out = partial;
  *splits_out = pl.splits;
  return run_plan(s, pl, P, dy, st);
}

}  // namespace dirb200
