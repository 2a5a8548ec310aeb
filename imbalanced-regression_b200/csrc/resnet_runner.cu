// Native runner of the bottleneck-ResNet backbone (agedb-dir/resnet.py:41-70,73-138): sequences the
// wgmma convolutions and the HBM-bound layers for one forward and one backward pass over a fixed
// batch shape, owning every activation / gradient / operand buffer (NHWC bf16) so that a training
// step issues no allocation and no host synchronisation.
//
// Parameters and their gradients live in ONE flat fp32 buffer each, laid out in the reference's
// named_parameters() order (conv1.weight, bn1.weight, bn1.bias, layer1.0.conv1.weight, ...), which the
// Python module (resnet.py) exposes as ordinary nn.Parameter views -> identical state_dict keys/shapes.
#include <stdlib.h>
#include <vector>
#include "common.cuh"
#include "conv.cuh"
#include "nn.cuh"

namespace dirb200 {

struct BNLayer {
  int c = 0;
  size_t gamma_off = 0, beta_off = 0;  // in the flat parameter buffer (floats)
  size_t rm_off = 0, rv_off = 0;       // in the flat BN running-statistics buffer (floats)
  float *mean = nullptr, *invstd = nullptr, *scale = nullptr, *shift = nullptr, *coef = nullptr;  // coef: [3][c] BN-backward
};

struct ConvLayer {
  ConvShape s{};
  bool stem = false;
  size_t w_off = 0;
  __nv_bfloat16 *wf = nullptr, *wd = nullptr;  // GEMM operands (fprop / dgrad layouts)
  float* wpart = nullptr;                      // split-K partials of this layer's weight gradient
  __nv_bfloat16* y = nullptr;                  // raw conv output [rows][cout]
  __nv_bfloat16* a = nullptr;                  // relu(bn(y)) when this conv is followed by BN+ReLU
  int64_t rows = 0;                            // n*ho*wo
  BNLayer bn;
};

struct Block {
  ConvLayer c1, c2, c3, ds;
  bool has_ds = false;
  const __nv_bfloat16* in = nullptr;
  __nv_bfloat16* out = nullptr;
  uint8_t* mask = nullptr;     // ReLU mask of `out`, 1 bit per element ([rows][c/8] bytes), for the backward pass
};

}  // namespace dirb200

using namespace dirb200;

struct dirb200_net {
  int n = 0, h = 0, w = 0;
  ConvLayer stem;
  std::vector<Block> blocks;
  __nv_bfloat16 *x_s2d = nullptr, *pool_out = nullptr;
  uint8_t* pool_idx = nullptr;
  int pool_h = 0, pool_w = 0;
  int feat_c = 0, feat_hw = 0;
  __nv_bfloat16* scratch[8] = {};
  WgradReduceDesc* reduce_descs = nullptr;     // device table, conv layers in backward-stage order
  std::vector<int> reduce_begin;               // first table entry of stage s (0 = stem, 1.. = layer groups); +1 sentinel
  float* bn_partial = nullptr;   // per-CTA partial sums of the BN column reductions (backward)
  float* stat_partial = nullptr; // per-CTA BN statistics [CTA][2][c] written by the conv fprop epilogue (conv.cuh)
  PrepDesc* prep_descs = nullptr; // device table for the single weight re-layout launch
  BnEvalDesc* bn_eval_descs = nullptr;  // device table: every BN layer, for the single eval-coefficient launch
  int num_bns = 0, max_bn_c = 0;
  int num_convs = 0;
  size_t param_count = 0, running_count = 0, activation_bytes = 0;
  std::vector<void*> allocs;
  bool forward_was_training = false;
  // backward runs stage by stage (layer4 .. layer1, stem) so that the caller can start the gradient all-reduce of a
  // finished stage while the earlier stages still compute; the incoming-gradient buffers live here between the calls
  std::vector<int> stage_begin;          // first block of stage s (1-based stages; stage_begin[num_stages+1] = #blocks)
  int bwd_next_stage = -1;               // stage the next dirb200_resnet_backward_stage call must name (-1: none pending)
  __nv_bfloat16 *bw_gA = nullptr, *bw_gB = nullptr, *bw_nA = nullptr, *bw_nB = nullptr, *bw_spareB = nullptr;
  int bw_gB_h = 0, bw_gB_w = 0;          // > 0: bw_gB is the compact [n, h/2, w/2, c] gradient of a stride-2 1x1 downsample
  // CUDA graphs of the launch sequences whose pointers never change (the training forward after the input re-layout,
  // every backward stage after the average-pool backward): captured on the second call, replayed from then on
  struct GraphSlot {
    cudaGraphExec_t exec = nullptr;
    const void *k0 = nullptr, *k1 = nullptr;   // the (params, running / grads) pointers the capture holds
    int warm = 0;
    int64_t launches = 0;                      // kernel launches inside (added to the launch counter per replay)
    // host-side state the captured calls leave behind (backward stages)
    __nv_bfloat16 *gA = nullptr, *gB = nullptr, *nA = nullptr, *nB = nullptr, *spareB = nullptr;
    int gB_h = 0, gB_w = 0;
  };
  GraphSlot g_fwd, g_bwd[6];
  // multi-scale (encoder) mode, dirb200_resnet_forward_blocks / dirb200_resnet_backward_blocks_stage: graphs of their
  // own.  A backward stage's sequence depends on the topmost stage that received a gradient (it fixes which scratch
  // buffers hold the incoming pair) and on whether the stage's own block gradient is added: [stage][top][d_block]
  GraphSlot g_fwd_blocks, g_bwd_blocks[6][6][2];
  bool bwd_blocks = false;   // the pending backward is the multi-scale one
  int bwd_top = -1;          // multi-scale backward: topmost stage that received a gradient so far (-1: none)
  cudaStream_t cap_stream = nullptr;               // capture happens on a private stream (the caller's may be the legacy default stream, which cannot capture)
  float *enc_buf = nullptr, *denc_buf = nullptr;   // fixed-address copies of the forward's output / the backward's input
  // optional per-kernel-class timing (CUDA events around every launch group)
  bool profiling = false;
  struct ProfRec { int kind; cudaEvent_t a, b; };
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> event_pool;
};

namespace dirb200 {

static bool dev_alloc(dirb200_net* net, void** p, size_t bytes) {
  if (cudaMalloc(p, bytes) != cudaSuccess) {
    set_error("resnet_create: cudaMalloc of %zu bytes failed", bytes);
    return false;
  }
  net->allocs.push_back(*p);
  net->activation_bytes += bytes;
  return true;
}

#define NET_ALLOC(ptr, bytes)                                                     \
  do {                                                                            \
    if (!dev_alloc(net, reinterpret_cast<void**>(&(ptr)), (bytes))) return false; \
  } while (0)

static bool setup_bn(dirb200_net* net, BNLayer& bn, int c) {
  bn.c = c;
  bn.gamma_off = net->param_count;
  bn.beta_off = net->param_count + c;
  net->param_count += 2 * (size_t)c;
  bn.rm_off = net->running_count;
  bn.rv_off = net->running_count + c;
  net->running_count += 2 * (size_t)c;
  float* f = nullptr;
  NET_ALLOC(f, sizeof(float) * 7 * c);
  bn.mean = f; bn.invstd = f + c; bn.scale = f + 2 * c; bn.shift = f + 3 * c; bn.coef = f + 4 * c;
  return true;
}

static bool setup_conv(dirb200_net* net, ConvLayer& cv, int n, int h, int w, int cin, int cout, int k, int stride,
                       int pad, bool stem, bool with_act) {
  cv.stem = stem;
  const int ho = (h + 2 * pad - k) / stride + 1, wo = (w + 2 * pad - k) / stride + 1;
  if (stem) cv.s = ConvShape{n, h / 2, w / 2, 16, cout, 4, 4, 1, 2, h / 2, w / 2};
  else cv.s = ConvShape{n, h, w, cin, cout, k, k, stride, pad, ho, wo};
  cv.w_off = net->param_count;
  net->param_count += (size_t)cout * cin * k * k;
  cv.rows = (int64_t)n * ho * wo;
  const size_t welems = stem ? (size_t)cout * 256 : (size_t)cout * cin * k * k;
  NET_ALLOC(cv.wf, welems * 2);
  if (!stem) NET_ALLOC(cv.wd, welems * 2);
  NET_ALLOC(cv.wpart, conv_wgrad_workspace_bytes(cv.s));
  NET_ALLOC(cv.y, (size_t)cv.rows * cout * 2);
  if (with_act) NET_ALLOC(cv.a, (size_t)cv.rows * cout * 2);
  return setup_bn(net, cv.bn, cout);
}

static bool build(dirb200_net* net, const int* blocks_per_stage, int num_stages) {
  const int n = net->n;
  // the stem's activation is never materialised: BN + ReLU are fused into the max pool (bn_relu_maxpool_fwd)
  if (!setup_conv(net, net->stem, n, net->h, net->w, 3, 64, 7, 2, 3, true, false)) return false;
  int h = net->h / 2, w = net->w / 2;
  NET_ALLOC(net->x_s2d, (size_t)n * h * w * 16 * 2);
  net->pool_h = (h - 1) / 2 + 1;
  net->pool_w = (w - 1) / 2 + 1;
  const size_t pool_elems = (size_t)n * net->pool_h * net->pool_w * 64;
  NET_ALLOC(net->pool_out, pool_elems * 2);
  NET_ALLOC(net->pool_idx, pool_elems);
  h = net->pool_h; w = net->pool_w;
  int inplanes = 64;
  const __nv_bfloat16* cur = net->pool_out;
  size_t max_act = (size_t)net->stem.rows * 64;
  net->stage_begin.assign(1, 0);
  for (int st = 0; st < num_stages; ++st) {
    const int planes = 64 << st;
    net->stage_begin.push_back((int)net->blocks.size());
    for (int b = 0; b < blocks_per_stage[st]; ++b) {
      const int stride = (b == 0 && st > 0) ? 2 : 1;
      net->blocks.emplace_back();
      Block& B = net->blocks.back();
      B.in = cur;
      B.has_ds = (b == 0) && (stride != 1 || inplanes != planes * 4);
      if (!setup_conv(net, B.c1, n, h, w, inplanes, planes, 1, 1, 0, false, true)) return false;
      if (!setup_conv(net, B.c2, n, h, w, planes, planes, 3, stride, 1, false, true)) return false;
      const int h2 = B.c2.s.ho, w2 = B.c2.s.wo;
      if (!setup_conv(net, B.c3, n, h2, w2, planes, planes * 4, 1, 1, 0, false, false)) return false;
      if (B.has_ds && !setup_conv(net, B.ds, n, h, w, inplanes, planes * 4, 1, stride, 0, false, false)) return false;
      NET_ALLOC(B.out, (size_t)B.c3.rows * planes * 4 * 2);
      NET_ALLOC(B.mask, (size_t)B.c3.rows * planes * 4 / 8);
      max_act = std::max(max_act, (size_t)B.c1.rows * std::max(inplanes, planes));
      max_act = std::max(max_act, (size_t)B.c3.rows * planes * 4);
      cur = B.out;
      inplanes = planes * 4;
      h = h2; w = w2;
    }
  }
  net->stage_begin.push_back((int)net->blocks.size());
  net->feat_c = inplanes;
  net->feat_hw = h * w;
  for (int i = 0; i < 8; ++i) NET_ALLOC(net->scratch[i], max_act * 2);
  {
    // split-K reduction jobs: every conv owns its partial buffer; one launch reduces a whole backward stage
    std::vector<WgradReduceDesc> rd;
    auto addr = [&](const ConvLayer& cv) {
      rd.push_back(WgradReduceDesc{cv.wpart, cv.w_off, conv_wgrad_splits(cv.s), cv.s.cout, cv.stem ? 3 : cv.s.cin,
                                   cv.stem ? 7 : cv.s.kh, cv.stem ? 7 : cv.s.kw, cv.stem ? 1 : 0});
    };
    net->reduce_begin.clear();
    net->reduce_begin.push_back(0);
    addr(net->stem);
    for (int stg = 1; stg <= num_stages; ++stg) {
      net->reduce_begin.push_back((int)rd.size());
      for (int bi = net->stage_begin[stg]; bi < net->stage_begin[stg + 1]; ++bi) {
        Block& B = net->blocks[bi];
        addr(B.c1); addr(B.c2); addr(B.c3);
        if (B.has_ds) addr(B.ds);
      }
    }
    net->reduce_begin.push_back((int)rd.size());
    NET_ALLOC(net->reduce_descs, sizeof(WgradReduceDesc) * rd.size());
    if (cudaMemcpy(net->reduce_descs, rd.data(), sizeof(WgradReduceDesc) * rd.size(), cudaMemcpyHostToDevice) != cudaSuccess)
      return false;
  }
  NET_ALLOC(net->enc_buf, sizeof(float) * (size_t)n * net->feat_c);
  NET_ALLOC(net->denc_buf, sizeof(float) * (size_t)n * net->feat_c);
  NET_ALLOC(net->bn_partial, sizeof(float) * bn_partial_floats(net->feat_c));
  NET_ALLOC(net->stat_partial, sizeof(float) * bn_partial_floats(net->feat_c));
  std::vector<PrepDesc> descs;
  auto add = [&](const ConvLayer& cv) {
    descs.push_back(make_prep_desc(cv.w_off, cv.s.cout, cv.stem ? 3 : cv.s.cin, cv.stem ? 7 : cv.s.kh, cv.stem ? 7 : cv.s.kw,
                                   cv.stem ? 1 : 0, cv.wf, cv.wd));
  };
  add(net->stem);
  for (Block& B : net->blocks) {
    add(B.c1); add(B.c2); add(B.c3);
    if (B.has_ds) add(B.ds);
  }
  net->num_convs = (int)descs.size();
  NET_ALLOC(net->prep_descs, sizeof(PrepDesc) * descs.size());
  if (cudaMemcpy(net->prep_descs, descs.data(), sizeof(PrepDesc) * descs.size(), cudaMemcpyHostToDevice) != cudaSuccess)
    return false;
  std::vector<BnEvalDesc> bd;
  auto addbn = [&](const BNLayer& bn) {
    bd.push_back(BnEvalDesc{bn.c, bn.gamma_off, bn.beta_off, bn.rm_off, bn.rv_off, bn.scale, bn.shift});
    net->max_bn_c = std::max(net->max_bn_c, bn.c);
  };
  addbn(net->stem.bn);
  for (Block& B : net->blocks) {
    addbn(B.c1.bn); addbn(B.c2.bn); addbn(B.c3.bn);
    if (B.has_ds) addbn(B.ds.bn);
  }
  net->num_bns = (int)bd.size();
  NET_ALLOC(net->bn_eval_descs, sizeof(BnEvalDesc) * bd.size());
  return cudaMemcpy(net->bn_eval_descs, bd.data(), sizeof(BnEvalDesc) * bd.size(), cudaMemcpyHostToDevice) == cudaSuccess;
}

#define RUN(expr)                    \
  do {                               \
    if (int _rc = (expr)) return _rc; \
  } while (0)

enum ProfKind { kPrep = 0, kFprop, kDgrad, kWgrad, kWgradReduce, kBnStats, kBnApply, kBnBwdReduce, kBnBwdApply, kPool,
                kNumProfKinds };

static cudaEvent_t prof_event(dirb200_net* net) {
  if (!net->event_pool.empty()) {
    cudaEvent_t e = net->event_pool.back();
    net->event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
static inline void prof_begin(dirb200_net* net, int kind, cudaStream_t st) {
  if (!net->profiling) return;
  dirb200_net::ProfRec r{kind, prof_event(net), prof_event(net)};
  cudaEventRecord(r.a, st);
  net->prof.push_back(r);
}
static inline void prof_end(dirb200_net* net, cudaStream_t st) {
  if (!net->profiling) return;
  cudaEventRecord(net->prof.back().b, st);
}
// RUN with the launch(es) attributed to a kernel class when profiling is on
#define RUNP(kind, expr)          \
  do {                            \
    prof_begin(net, (kind), st);  \
    int _rc = (expr);             \
    prof_end(net, st);            \
    if (_rc) return _rc;          \
  } while (0)

// DIRB200_FUSED_STATS=0: batch statistics by the separate bn_stats pass over y (A/B measurements) instead of the
// conv epilogue.
static bool fused_stats() {
  static const bool on = [] {
    const char* e = getenv("DIRB200_FUSED_STATS");
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}

static int conv_bn_forward(dirb200_net* net, ConvLayer& cv, const __nv_bfloat16* in, const float* params,
                           float* running, bool training, cudaStream_t st) {
  BNLayer& bn = cv.bn;
  if (training) {
    // batch statistics come out of the conv epilogue (per-CTA column sums of the rounded outputs): y is not re-read
    StatLayout lay{};
    const bool fused = fused_stats();
    RUNP(kFprop, conv_fprop(in, cv.wf, cv.y, cv.s, cv.stem, st, fused ? net->stat_partial : nullptr, &lay));
    if (!fused) {
      int nblk = 0;
      RUNP(kBnStats, bn_stats(cv.y, cv.rows, bn.c, net->stat_partial, &nblk, st));
      lay = StatLayout{nblk, 1, bn.c, 1};
    }
    RUNP(kBnStats, bn_finalize(net->stat_partial, lay, cv.rows, bn.c, params + bn.gamma_off, params + bn.beta_off, 1e-5f,
                               0.1f, running ? running + bn.rm_off : nullptr, running ? running + bn.rv_off : nullptr,
                               bn.mean, bn.invstd, bn.scale, bn.shift, st));
  } else {
    RUNP(kFprop, conv_fprop(in, cv.wf, cv.y, cv.s, cv.stem, st));
    RUNP(kBnStats, bn_eval_coeffs(bn.c, params + bn.gamma_off, params + bn.beta_off, 1e-5f, running + bn.rm_off,
                                  running + bn.rv_off, bn.scale, bn.shift, st));
  }
  if (cv.a)
    RUNP(kBnApply, bn_apply(cv.y, bn.scale, bn.shift, nullptr, nullptr, nullptr, nullptr, true, cv.rows, bn.c, cv.a, nullptr, st));
  return DIRB200_OK;
}

// weight-gradient GEMM of one conv into its own split-K partial buffer; the reduction into the flat gradient happens
// once per backward stage (wgrad_reduce_stage)
static int wgrad_step(dirb200_net* net, const __nv_bfloat16* x, const __nv_bfloat16* dy, ConvLayer& cv, cudaStream_t st) {
  int splits = 1;
  RUNP(kWgrad, conv_wgrad_partials(x, dy, cv.wpart, cv.s, cv.stem, &splits, st));
  return DIRB200_OK;
}

static int wgrad_reduce_stage(dirb200_net* net, int stage, float* grads, cudaStream_t st) {
  const int lo = net->reduce_begin[stage], hi = net->reduce_begin[stage + 1];
  RUNP(kWgradReduce, wgrad_reduce_all(net->reduce_descs + lo, hi - lo, grads, st));
  return DIRB200_OK;
}

// BN backward for a conv followed by BN+ReLU: g = d loss / d relu-output.  The ReLU mask is re-derived from
// (y, scale, shift): the activation cv.a is not read.
// moments: the layout of the (sum dz, sum dz*y) rows the dgrad that PRODUCED g already accumulated in its epilogue
// (dgrad_with_bn_moments below) -- then the bn_bwd_reduce pass over (g, y) is skipped.
static int conv_bn_backward(dirb200_net* net, ConvLayer& cv, const __nv_bfloat16* g, const float* params, float* grads,
                            __nv_bfloat16* dy, cudaStream_t st, const StatLayout* moments = nullptr) {
  BNLayer& bn = cv.bn;
  if (moments) {
    RUNP(kBnBwdApply, bn_bwd_coeffs_layout(net->bn_partial, *moments, cv.rows, bn.c, bn.mean, bn.invstd,
                                           params + bn.gamma_off, grads + bn.gamma_off, grads + bn.beta_off, bn.coef, st));
  } else {
    int nblk = 0;
    RUNP(kBnBwdReduce, bn_bwd_reduce(g, nullptr, cv.y, nullptr, bn.scale, bn.shift, nullptr, cv.rows, bn.c,
                                     net->bn_partial, &nblk, st));
    RUNP(kBnBwdApply, bn_bwd_coeffs(net->bn_partial, nblk, 2, 1, cv.rows, bn.c, bn.mean, bn.invstd,
                                    params + bn.gamma_off, grads + bn.gamma_off, grads + bn.beta_off, bn.coef, st));
  }
  RUNP(kBnBwdApply, bn_bwd_apply(g, nullptr, cv.y, bn.coef, nullptr, nullptr, bn.scale, bn.shift, nullptr, cv.rows, bn.c,
                                 dy, nullptr, nullptr, st));
  return DIRB200_OK;
}

// Inference forward (agedb-dir/train.py:286-335 validate(); resnet.py:46-66,128-138 under model.eval()): BatchNorm uses
// the running statistics, so it is a per-channel affine map that folds into the conv epilogue -- every
// conv -> BN [-> ReLU] and the whole conv3 -> BN -> (+ shortcut) -> ReLU tail of a block is ONE launch, and no raw conv
// output is written.  ~58 launches instead of ~165.  DIRB200_FOLDED_EVAL=0 keeps the unfused sequence (A/B checks).
static bool folded_eval() {
  static const bool on = [] {
    const char* e = getenv("DIRB200_FOLDED_EVAL");
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}

// enc_out == nullptr: no average pool (multi-scale mode reads the block outputs)
static int forward_eval_folded(dirb200_net* net, const float* params, const float* running, float* enc_out,
                               cudaStream_t st) {
  RUNP(kBnStats, bn_eval_coeffs_all(net->bn_eval_descs, net->num_bns, net->max_bn_c, params, running, 1e-5f, st));
  // stem: plain conv, then BN + ReLU inside the max pool (as in training; the activation is never materialised)
  RUNP(kFprop, conv_fprop(net->x_s2d, net->stem.wf, net->stem.y, net->stem.s, true, st));
  RUNP(kPool, bn_relu_maxpool_fwd(net->stem.y, net->stem.bn.scale, net->stem.bn.shift, net->n, net->stem.s.ho,
                                  net->stem.s.wo, 64, net->pool_out, net->pool_idx, st));
  for (Block& B : net->blocks) {
    RUNP(kFprop, conv_fprop_affine(B.in, B.c1.wf, B.c1.a, B.c1.s, ConvEpilogue{B.c1.bn.scale, B.c1.bn.shift, nullptr, true}, st));
    RUNP(kFprop, conv_fprop_affine(B.c1.a, B.c2.wf, B.c2.a, B.c2.s, ConvEpilogue{B.c2.bn.scale, B.c2.bn.shift, nullptr, true}, st));
    const __nv_bfloat16* shortcut = B.in;
    if (B.has_ds) {
      RUNP(kFprop, conv_fprop_affine(B.in, B.ds.wf, B.ds.y, B.ds.s, ConvEpilogue{B.ds.bn.scale, B.ds.bn.shift, nullptr, false}, st));
      shortcut = B.ds.y;
    }
    RUNP(kFprop, conv_fprop_affine(B.c2.a, B.c3.wf, B.out, B.c3.s, ConvEpilogue{B.c3.bn.scale, B.c3.bn.shift, shortcut, true}, st));
  }
  if (enc_out) RUNP(kPool, avgpool_fwd(net->blocks.back().out, net->n, net->feat_hw, net->feat_c, enc_out, st));
  return DIRB200_OK;
}

// The launch sequence of a forward after the input re-layout (training: batch statistics; else the unfused eval form).
// enc_out == nullptr: no average pool.
static int forward_body(dirb200_net* net, const float* params, float* running, bool tr, float* enc_out,
                        cudaStream_t st) {
  RUN(conv_bn_forward(net, net->stem, net->x_s2d, params, running, tr, st));       // stem.a == nullptr: no bn_apply
  RUNP(kPool, bn_relu_maxpool_fwd(net->stem.y, net->stem.bn.scale, net->stem.bn.shift, net->n, net->stem.s.ho,
                                  net->stem.s.wo, 64, net->pool_out, net->pool_idx, st));
  for (Block& B : net->blocks) {
    RUN(conv_bn_forward(net, B.c1, B.in, params, running, tr, st));
    RUN(conv_bn_forward(net, B.c2, B.c1.a, params, running, tr, st));
    RUN(conv_bn_forward(net, B.c3, B.c2.a, params, running, tr, st));
    if (B.has_ds) {
      RUN(conv_bn_forward(net, B.ds, B.in, params, running, tr, st));
      RUNP(kBnApply, bn_apply(B.c3.y, B.c3.bn.scale, B.c3.bn.shift, nullptr, B.ds.y, B.ds.bn.scale, B.ds.bn.shift, true,
                              B.c3.rows, B.c3.bn.c, B.out, tr ? B.mask : nullptr, st));
    } else {
      RUNP(kBnApply, bn_apply(B.c3.y, B.c3.bn.scale, B.c3.bn.shift, B.in, nullptr, nullptr, nullptr, true, B.c3.rows,
                              B.c3.bn.c, B.out, tr ? B.mask : nullptr, st));
    }
  }
  if (enc_out) RUNP(kPool, avgpool_fwd(net->blocks.back().out, net->n, net->feat_hw, net->feat_c, enc_out, st));
  return DIRB200_OK;
}

// Multi-scale mode hands out (and takes a gradient for) the output of the last block of every layer group; that block
// must be an identity block (true of every layer group of ResNet-50 and deeper), whose output BN-backward reduction
// takes the group's gradient as a third operand.
static int check_blocks_mode(const dirb200_net* net, const char* who) {
  const int nst = (int)net->stage_begin.size() - 2;
  for (int s = 1; s <= nst; ++s)
    DIRB_CHECK_ARG(!net->blocks[net->stage_begin[s + 1] - 1].has_ds,
                   "%s: layer group %d ends in a downsample block; multi-scale mode needs an identity block there", who, s);
  return DIRB200_OK;
}

// The fixed-pointer launch sequences of a training step (~390 of its ~410 launches) are replayed as CUDA graphs (see
// GraphSlot), which removes the dependent-launch gaps of a stream (A/B on an H100 80GB HBM3 at a 400 W power limit,
// bench.py batch 256, two runs each: 41.6 ms per step with graphs, 42.1 ms eager).  DIRB200_GRAPH=0 launches eagerly.
static bool graphs_enabled() {
  static const bool on = [] {
    const char* e = getenv("DIRB200_GRAPH");
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}

// Runs `body(st)` -- a sequence of launches that depends on nothing but (k0, k1) and the net's own buffers -- eagerly
// the first time (also the one-time kernel attribute calls), captures it the second time, replays it afterwards.
template <typename F>
static int run_graphed(dirb200_net* net, dirb200_net::GraphSlot& g, const void* k0, const void* k1, cudaStream_t st,
                       F&& body) {
  if (!graphs_enabled() || net->profiling) return body(st);
  if (g.exec && g.k0 == k0 && g.k1 == k1) {
    DIRB_CUDA(cudaGraphLaunch(g.exec, st));
    g_launches.fetch_add(g.launches);
    return DIRB200_OK;
  }
  if (g.exec) {
    cudaGraphExecDestroy(g.exec);
    g.exec = nullptr;
    g.warm = 0;
  }
  if (g.warm == 0 || g.k0 != k0 || g.k1 != k1) {
    g.k0 = k0; g.k1 = k1; g.warm = 1;
    return body(st);
  }
  const int64_t before = g_launches.load();
  if (!net->cap_stream) DIRB_CUDA(cudaStreamCreateWithFlags(&net->cap_stream, cudaStreamNonBlocking));
  DIRB_CUDA(cudaStreamBeginCapture(net->cap_stream, cudaStreamCaptureModeThreadLocal));
  const int rc = body(net->cap_stream);
  cudaGraph_t graph = nullptr;
  const cudaError_t e = cudaStreamEndCapture(net->cap_stream, &graph);
  if (rc != DIRB200_OK || e != cudaSuccess || graph == nullptr) {
    if (graph) cudaGraphDestroy(graph);
    if (rc == DIRB200_OK) set_error("resnet: stream capture failed (%s)", cudaGetErrorString(e));
    (void)cudaGetLastError();
    return rc != DIRB200_OK ? rc : DIRB200_ERR_CUDA;
  }
  g.launches = g_launches.load() - before;
  g_launches.fetch_sub(g.launches);                // nothing ran yet
  const cudaError_t ei = cudaGraphInstantiate(&g.exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ei != cudaSuccess) {
    g.exec = nullptr;
    set_error("resnet: cudaGraphInstantiate failed (%s)", cudaGetErrorString(ei));
    return DIRB200_ERR_CUDA;
  }
  DIRB_CUDA(cudaGraphLaunch(g.exec, st));
  g_launches.fetch_add(g.launches);
  return DIRB200_OK;
}

// DIRB200_FUSED_BWD_MOMENTS=0: separate bn_bwd_reduce passes everywhere (A/B measurements).
static bool fused_bwd_moments() {
  static const bool on = [] {
    const char* e = getenv("DIRB200_FUSED_BWD_MOMENTS");
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}

// dgrad of `cv` whose output g is the gradient w.r.t. relu(bn(prev.y)): where the kernel can, the BN-backward moments of
// `prev` come out of the epilogue (*fused = true, *lay = their row layout in net->bn_partial)
static int dgrad_with_bn_moments(dirb200_net* net, const __nv_bfloat16* dy, ConvLayer& cv, ConvLayer& prev,
                                 __nv_bfloat16* g, StatLayout* lay, bool* fused, cudaStream_t st) {
  *fused = fused_bwd_moments() && conv_dgrad_fuses_bn_moments(cv.s);
  if (!*fused) {
    RUNP(kDgrad, conv_dgrad(dy, cv.wd, g, cv.s, st));
    return DIRB200_OK;
  }
  const DgradBnMoments bm{prev.y, prev.bn.scale, prev.bn.shift, net->bn_partial, lay};
  RUNP(kDgrad, conv_dgrad(dy, cv.wd, g, cv.s, st, &bm));
  return DIRB200_OK;
}

}  // namespace dirb200

// bounds of the packed pixel coordinates of the convolutions (see dirb200_resnet_create)
static constexpr int kMaxNetBatch = 1 << 13;        // image index: 13 bits
static constexpr int kMaxNetSide = 2 * (1 << 9);    // stem-output row / column: 9 bits, the stem halves H and W

extern "C" {

int dirb200_resnet_create(int n, int h, int w, const int* blocks_per_stage, int num_stages, dirb200_net** out) {
  DIRB_CHECK_ARG(out && blocks_per_stage && n > 0 && num_stages >= 1 && num_stages <= 4, "resnet_create: bad arguments");
  // the input space-to-depth needs even H and W, the max-pool backward an even stem output (H/2, W/2)
  DIRB_CHECK_ARG(h > 0 && w > 0 && h % 4 == 0 && w % 4 == 0, "resnet_create: H and W must be multiples of 4 (got %dx%d)",
                 h, w);
  // the implicit-GEMM convolutions pack a pixel of the largest map they index (the stem output, H/2 x W/2) as
  // image (13 bits) | row (9 bits) | column (9 bits) (conv_igemm.cu, pack_pixel / row_pre), and that map must hold
  // fewer than 2^31 pixels
  DIRB_CHECK_ARG(n <= kMaxNetBatch, "resnet_create: N must be at most %d (got %d)", kMaxNetBatch, n);
  DIRB_CHECK_ARG(h <= kMaxNetSide && w <= kMaxNetSide, "resnet_create: H and W must be at most %d (got %dx%d)", kMaxNetSide,
                 h, w);
  DIRB_CHECK_ARG((int64_t)n * (h / 2) * (w / 2) < (int64_t(1) << 31),
                 "resnet_create: N * H/2 * W/2 must be below 2^31 (got %d x %d x %d)", n, h / 2, w / 2);
  dirb200_net* net = new dirb200_net();
  net->n = n; net->h = h; net->w = w;
  if (!build(net, blocks_per_stage, num_stages)) {
    for (void* p : net->allocs) cudaFree(p);
    delete net;
    return DIRB200_ERR_CUDA;
  }
  *out = net;
  return DIRB200_OK;
}

void dirb200_resnet_destroy(dirb200_net* net) {
  if (!net) return;
  if (net->cap_stream) cudaStreamDestroy(net->cap_stream);
  if (net->g_fwd.exec) cudaGraphExecDestroy(net->g_fwd.exec);
  if (net->g_fwd_blocks.exec) cudaGraphExecDestroy(net->g_fwd_blocks.exec);
  for (auto& g : net->g_bwd)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  for (auto& per_stage : net->g_bwd_blocks)
    for (auto& per_top : per_stage)
      for (auto& g : per_top)
        if (g.exec) cudaGraphExecDestroy(g.exec);
  for (void* p : net->allocs) cudaFree(p);
  delete net;
}

int64_t dirb200_resnet_param_count(const dirb200_net* net) { return net ? (int64_t)net->param_count : -1; }
int64_t dirb200_resnet_running_count(const dirb200_net* net) { return net ? (int64_t)net->running_count : -1; }
int64_t dirb200_resnet_feature_dim(const dirb200_net* net) { return net ? net->feat_c : -1; }
int64_t dirb200_resnet_device_bytes(const dirb200_net* net) { return net ? (int64_t)net->activation_bytes : -1; }

/* Per-kernel-class device timing (CUDA events around every launch group of forward/backward).
 * Classes: 0 prep (weight re-layout, s2d), 1 conv fprop, 2 conv dgrad, 3 conv wgrad GEMM, 4 wgrad split-K reduce,
 * 5 BN statistics, 6 BN apply, 7 BN backward reduce, 8 BN backward apply, 9 pooling. */
int dirb200_resnet_set_profiling(dirb200_net* net, int enabled) {
  DIRB_CHECK_ARG(net, "resnet_set_profiling: null net");
  net->profiling = enabled != 0;
  return DIRB200_OK;
}

/* Synchronises, sums the recorded intervals per class into ms_by_kind[10] / launches_by_kind[10], clears the log. */
int dirb200_resnet_read_profile(dirb200_net* net, double* ms_by_kind, int64_t* groups_by_kind) {
  DIRB_CHECK_ARG(net && ms_by_kind && groups_by_kind, "resnet_read_profile: null pointer");
  for (int i = 0; i < kNumProfKinds; ++i) { ms_by_kind[i] = 0.0; groups_by_kind[i] = 0; }
  for (auto& r : net->prof) {
    DIRB_CUDA(cudaEventSynchronize(r.b));
    float ms = 0.f;
    DIRB_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
    ms_by_kind[r.kind] += ms;
    groups_by_kind[r.kind] += 1;
    net->event_pool.push_back(r.a);
    net->event_pool.push_back(r.b);
  }
  net->prof.clear();
  return DIRB200_OK;
}

/* x fp32 NCHW [n,3,h,w] -> enc fp32 [n, feature_dim]  (conv1 ... avgpool + view, resnet.py:128-138).
 * training != 0: batch statistics, running statistics updated (momentum 0.1); else running statistics. */
int dirb200_resnet_forward(dirb200_net* net, const float* x_nchw, const float* params, float* bn_running, int training,
                           float* enc_out, void* stream) {
  DIRB_CHECK_ARG(net && x_nchw && params && enc_out, "resnet_forward: null pointer");
  DIRB_CHECK_ARG(training || bn_running, "resnet_forward: eval mode needs the running statistics");
  cudaStream_t st = as_stream(stream);
  const bool tr = training != 0;
  RUNP(kPrep, prep_weights_all(params, net->prep_descs, net->num_convs, st));
  RUNP(kPrep, input_to_s2d(x_nchw, net->n, net->h, net->w, net->x_s2d, st));
  if (!tr && folded_eval()) {
    RUN(forward_eval_folded(net, params, bn_running, enc_out, st));
    net->forward_was_training = false;
    return DIRB200_OK;
  }
  const bool graphed = tr && graphs_enabled() && !net->profiling;
  float* enc_dst = graphed ? net->enc_buf : enc_out;
  auto body = [&](cudaStream_t st) -> int { return forward_body(net, params, bn_running, tr, enc_dst, st); };
  if (graphed) {
    RUN(run_graphed(net, net->g_fwd, params, bn_running, st, body));
    DIRB_CUDA(cudaMemcpyAsync(enc_out, net->enc_buf, sizeof(float) * (size_t)net->n * net->feat_c,
                              cudaMemcpyDeviceToDevice, st));
  } else {
    RUN(body(st));
  }
  net->forward_was_training = tr;
  return DIRB200_OK;
}

/* The same forward without the average pool (nyud2-dir/models/modules.py:33-58, E_resnet.forward): the output of the
 * last block of layer group s+1 goes to block_out[s], NHWC bf16 [n, h_s, w_s, C_s].  training == 0: the folded-BN
 * inference forward.  The training launch sequence is graph-replayed (a graph of its own) and the outputs are copied
 * out after it, so the caller's pointers may change from call to call. */
int dirb200_resnet_forward_blocks(dirb200_net* net, const float* x_nchw, const float* params, float* bn_running,
                                  int training, void* const* block_out, void* stream) {
  DIRB_CHECK_ARG(net && x_nchw && params && block_out, "resnet_forward_blocks: null pointer");
  DIRB_CHECK_ARG(training || bn_running, "resnet_forward_blocks: eval mode needs the running statistics");
  const int nst = (int)net->stage_begin.size() - 2;
  for (int s = 0; s < nst; ++s) DIRB_CHECK_ARG(block_out[s], "resnet_forward_blocks: null block_out[%d]", s);
  RUN(check_blocks_mode(net, "resnet_forward_blocks"));
  cudaStream_t st = as_stream(stream);
  const bool tr = training != 0;
  RUNP(kPrep, prep_weights_all(params, net->prep_descs, net->num_convs, st));
  RUNP(kPrep, input_to_s2d(x_nchw, net->n, net->h, net->w, net->x_s2d, st));
  if (!tr && folded_eval()) {
    RUN(forward_eval_folded(net, params, bn_running, nullptr, st));
  } else {
    auto body = [&](cudaStream_t st) -> int { return forward_body(net, params, bn_running, tr, nullptr, st); };
    if (tr) RUN(run_graphed(net, net->g_fwd_blocks, params, bn_running, st, body));
    else RUN(body(st));
  }
  for (int s = 0; s < nst; ++s) {
    const Block& B = net->blocks[net->stage_begin[s + 2] - 1];
    DIRB_CUDA(cudaMemcpyAsync(block_out[s], B.out, sizeof(__nv_bfloat16) * (size_t)B.c3.rows * B.c3.s.cout,
                              cudaMemcpyDeviceToDevice, st));
  }
  net->forward_was_training = tr;
  return DIRB200_OK;
}

}  // extern "C"

namespace dirb200 {

// blocks [lo, hi) in reverse order; the incoming gradient pair is net->bw_gA / bw_gB, plus g3 (may be null) for the
// output of block hi-1 (multi-scale mode: the gradient of a layer group's output from outside the network)
static int backward_blocks(dirb200_net* net, int lo, int hi, const float* params, float* grads, cudaStream_t st,
                           const __nv_bfloat16* g3 = nullptr) {
  __nv_bfloat16 *gA = net->bw_gA, *gB = net->bw_gB, *nA = net->bw_nA, *nB = net->bw_nB, *spareB = net->bw_spareB;
  __nv_bfloat16 *t1 = net->scratch[4], *t2 = net->scratch[5], *t3 = net->scratch[6];
  int gB_h = net->bw_gB_h, gB_w = net->bw_gB_w;
  for (int bi = hi - 1; bi >= lo; --bi) {
    Block& B = net->blocks[bi];
    BNLayer& b3 = B.c3.bn;
    // ---- block output: out = relu(bn3(y3) + identity); dz = (gA + gB) * (out > 0)
    int nblk = 0;
    const int kparts = B.has_ds ? 3 : 2;
    // identity blocks: the reduction also stores dz (= the gradient of the shortcut path, nB) so that the apply pass
    // reads ONE gradient tensor instead of gA, gB and the mask again
    RUNP(kBnBwdReduce, bn_bwd_reduce(gA, gB, B.c3.y, B.has_ds ? B.ds.y : nullptr, nullptr, nullptr, B.mask, B.c3.rows,
                                     b3.c, net->bn_partial, &nblk, st, gB_h, gB_w, B.has_ds ? nullptr : nB,
                                     bi == hi - 1 ? g3 : nullptr));
    if (B.has_ds) {
      BNLayer& bd = B.ds.bn;
      RUNP(kBnBwdApply, bn_bwd_coeffs(net->bn_partial, nblk, kparts, 2, B.c3.rows, b3.c, bd.mean, bd.invstd,
                                      params + bd.gamma_off, grads + bd.gamma_off, grads + bd.beta_off, bd.coef, st));
    }
    RUNP(kBnBwdApply, bn_bwd_coeffs(net->bn_partial, nblk, kparts, 1, B.c3.rows, b3.c, b3.mean, b3.invstd,
                                    params + b3.gamma_off, grads + b3.gamma_off, grads + b3.beta_off, b3.coef, st));
    if (B.has_ds)
      RUNP(kBnBwdApply, bn_bwd_apply(gA, gB, B.c3.y, b3.coef, B.ds.y, B.ds.bn.coef, nullptr, nullptr, B.mask, B.c3.rows,
                                     b3.c, t1, t2, nullptr, st, gB_h, gB_w));
    else
      RUNP(kBnBwdApply, bn_bwd_apply(nB, nullptr, B.c3.y, b3.coef, nullptr, nullptr, nullptr, nullptr, nullptr, B.c3.rows,
                                     b3.c, t1, nullptr, nullptr, st));
    gB_h = gB_w = 0;
    // ---- conv3
    RUN(wgrad_step(net, B.c2.a, t1, B.c3, st));
    StatLayout mlay{};
    bool mfused = false;
    RUN(dgrad_with_bn_moments(net, t1, B.c3, B.c2, t3, &mlay, &mfused, st));
    // ---- bn2 + conv2
    RUN(conv_bn_backward(net, B.c2, t3, params, grads, t1, st, mfused ? &mlay : nullptr));
    RUN(wgrad_step(net, B.c1.a, t1, B.c2, st));
    RUN(dgrad_with_bn_moments(net, t1, B.c2, B.c1, t3, &mlay, &mfused, st));
    // ---- bn1 + conv1
    RUN(conv_bn_backward(net, B.c1, t3, params, grads, t1, st, mfused ? &mlay : nullptr));
    RUN(wgrad_step(net, B.in, t1, B.c1, st));
    RUNP(kDgrad, conv_dgrad(t1, B.c1.wd, nA, B.c1.s, st));
    // ---- downsample branch
    if (B.has_ds) {
      RUN(wgrad_step(net, B.in, t2, B.ds, st));
      const ConvShape& d = B.ds.s;
      if (d.stride == 2 && d.kh == 1 && d.kw == 1 && d.pad == 0 && d.h % 2 == 0 && d.w % 2 == 0 && bi > 0 &&
          !net->blocks[bi - 1].has_ds) {
        // stride-2 1x1 downsample: its input gradient is non-zero at the even pixels only -> keep it COMPACT
        // ([n, h/2, w/2, cin], a plain GEMM over the strided grid); the previous block's output BN backward adds it at
        // the even positions (no memset of the full map, no scattered store, no dense re-reads of zeros)
        const ConvShape cs{d.n, d.ho, d.wo, d.cin, d.cout, 1, 1, 1, 0, d.ho, d.wo};
        RUNP(kDgrad, conv_dgrad(t2, B.ds.wd, nB, cs, st));
        gB_h = d.h;
        gB_w = d.w;
      } else {
        RUNP(kDgrad, conv_dgrad(t2, B.ds.wd, nB, B.ds.s, st));
      }
    }
    // the two gradients w.r.t. this block's input become the next (earlier) block's incoming pair
    __nv_bfloat16* oldA = gA;
    __nv_bfloat16* oldB = gB ? gB : spareB;
    gA = nA; gB = nB;
    nA = oldA; nB = oldB;
    spareB = nullptr;
  }
  net->bw_gA = gA; net->bw_gB = gB; net->bw_nA = nA; net->bw_nB = nB; net->bw_spareB = spareB;
  net->bw_gB_h = gB_h; net->bw_gB_w = gB_w;
  return DIRB200_OK;
}

// The work of one backward stage (the incoming gradients are in place), graph-replayed in slot g.  The captured
// sequence leaves host-side state behind (which scratch buffers hold the gradients entering the next stage): recorded
// at capture, restored at replay -- the sequence of buffers is the same in every step that uses the slot.
static int backward_stage_run(dirb200_net* net, int stage, const float* params, float* grads, const __nv_bfloat16* g3,
                              dirb200_net::GraphSlot& g, cudaStream_t st) {
  auto body = [&](cudaStream_t st) -> int {
    if (stage >= 1) {
      RUN(backward_blocks(net, net->stage_begin[stage], net->stage_begin[stage + 1], params, grads, st, g3));
    } else {
      // ---- stem: maxpool -> bn1+relu -> conv1 (no data gradient needed)
      __nv_bfloat16 *t1 = net->scratch[4], *t3 = net->scratch[6];
      RUNP(kPool, maxpool_bwd(net->bw_gA, net->bw_gB, net->pool_idx, net->n, net->stem.s.ho, net->stem.s.wo, 64, t3, st));
      RUN(conv_bn_backward(net, net->stem, t3, params, grads, t1, st));
      RUN(wgrad_step(net, net->x_s2d, t1, net->stem, st));
    }
    RUN(wgrad_reduce_stage(net, stage, grads, st));
    return DIRB200_OK;
  };
  if (!graphs_enabled() || net->profiling) return body(st);
  const bool replay = g.exec && g.k0 == params && g.k1 == grads;
  RUN(run_graphed(net, g, params, grads, st, body));
  if (replay) {
    net->bw_gA = g.gA; net->bw_gB = g.gB; net->bw_nA = g.nA; net->bw_nB = g.nB; net->bw_spareB = g.spareB;
    net->bw_gB_h = g.gB_h; net->bw_gB_w = g.gB_w;
  } else {
    g.gA = net->bw_gA; g.gB = net->bw_gB; g.nA = net->bw_nA; g.nB = net->bw_nB; g.spareB = net->bw_spareB;
    g.gB_h = net->bw_gB_h; g.gB_w = net->bw_gB_w;
  }
  return DIRB200_OK;
}

}  // namespace dirb200

extern "C" {

/* One stage of the backward pass: stage = number of stages (4 for ResNet-50) first -- average-pool backward of
 * d_enc and the last layer group --, then stage-1 ... 1 (layer groups), finally 0 (max-pool, stem BN, conv1).  Calls
 * must come in exactly that order after a training-mode forward; each ACCUMULATES the parameter gradients of its own
 * stage into grads (flat fp32, same layout as params), whose range dirb200_resnet_stage_param_range reports -- a
 * finished range can be all-reduced while the remaining stages run (agedb-dir/train.py:143,261: DataParallel's
 * gradient reduction, here overlapped).  d_enc is only read by the first call. */
int dirb200_resnet_backward_stage(dirb200_net* net, int stage, const float* d_enc, const float* params, float* grads,
                                  void* stream) {
  DIRB_CHECK_ARG(net && params && grads, "resnet_backward_stage: null pointer");
  const int nst = (int)net->stage_begin.size() - 2;
  DIRB_CHECK_ARG(stage >= 0 && stage <= nst, "resnet_backward_stage: bad stage %d", stage);
  cudaStream_t st = as_stream(stream);
  if (stage == nst) {
    DIRB_CHECK_ARG(net->forward_was_training, "resnet_backward: needs a preceding training-mode forward");
    DIRB_CHECK_ARG(d_enc, "resnet_backward_stage: the first stage needs d_enc");
    net->bw_gA = net->scratch[0]; net->bw_gB = nullptr; net->bw_nA = net->scratch[2]; net->bw_nB = net->scratch[3];
    net->bw_spareB = net->scratch[1];
    net->bw_gB_h = net->bw_gB_w = 0;
    RUNP(kPool, avgpool_bwd(d_enc, net->n, net->feat_hw, net->feat_c, net->bw_gA, st));
  } else {
    DIRB_CHECK_ARG(net->bwd_next_stage == stage && !net->bwd_blocks,
                   "resnet_backward_stage: stage %d out of order (expected %d%s)", stage, net->bwd_next_stage,
                   net->bwd_blocks ? " of a multi-scale backward" : "");
  }
  net->bwd_next_stage = -1;
  net->bwd_blocks = false;
  RUN(backward_stage_run(net, stage, params, grads, nullptr, net->g_bwd[stage], st));
  net->bwd_next_stage = stage - 1;          // -1 after the stem: nothing pending
  return DIRB200_OK;
}

/* Multi-scale backward (nyud2-dir/models/modules.py:33-58, E_resnet.forward): stage = num_stages first, then
 * num_stages-1 ... 1, then 0, after a training-mode forward.  Stage s >= 1 reads d_block, the bf16 NHWC gradient of
 * the output of layer group s (NULL: zero); stage 0 reads nothing.  A stage that receives no gradient, neither its own
 * nor from the stages above, does nothing: its parameter gradients keep their values. */
int dirb200_resnet_backward_blocks_stage(dirb200_net* net, int stage, const void* d_block, const float* params,
                                         float* grads, void* stream) {
  DIRB_CHECK_ARG(net && params && grads, "resnet_backward_blocks_stage: null pointer");
  const int nst = (int)net->stage_begin.size() - 2;
  DIRB_CHECK_ARG(stage >= 0 && stage <= nst, "resnet_backward_blocks_stage: bad stage %d", stage);
  DIRB_CHECK_ARG(stage > 0 || !d_block, "resnet_backward_blocks_stage: stage 0 (the stem) takes no block gradient");
  RUN(check_blocks_mode(net, "resnet_backward_blocks_stage"));
  cudaStream_t st = as_stream(stream);
  if (stage == nst) {
    DIRB_CHECK_ARG(net->forward_was_training, "resnet_backward_blocks_stage: needs a preceding training-mode forward");
    net->bwd_top = -1;
  } else {
    DIRB_CHECK_ARG(net->bwd_next_stage == stage && net->bwd_blocks,
                   "resnet_backward_blocks_stage: stage %d out of order (expected %d%s)", stage, net->bwd_next_stage,
                   net->bwd_blocks ? "" : " of a multi-scale backward");
  }
  net->bwd_next_stage = -1;
  net->bwd_blocks = true;
  const __nv_bfloat16* g3 = nullptr;
  if (stage > 0 && d_block) {
    const Block& B = net->blocks[net->stage_begin[stage + 1] - 1];
    const size_t bytes = sizeof(__nv_bfloat16) * (size_t)B.c3.rows * B.c3.s.cout;
    if (net->bwd_top < 0) {
      // the first gradient of this backward: it enters like the average-pool backward's output does
      net->bwd_top = stage;
      net->bw_gA = net->scratch[0]; net->bw_gB = nullptr; net->bw_nA = net->scratch[2]; net->bw_nB = net->scratch[3];
      net->bw_spareB = net->scratch[1];
      net->bw_gB_h = net->bw_gB_w = 0;
      DIRB_CUDA(cudaMemcpyAsync(net->bw_gA, d_block, bytes, cudaMemcpyDeviceToDevice, st));
    } else {
      // a third operand of the group output's BN-backward reduction, staged at a fixed address for the graph
      DIRB_CUDA(cudaMemcpyAsync(net->scratch[7], d_block, bytes, cudaMemcpyDeviceToDevice, st));
      g3 = net->scratch[7];
    }
  }
  if (net->bwd_top >= 0)
    RUN(backward_stage_run(net, stage, params, grads, g3, net->g_bwd_blocks[stage][net->bwd_top][g3 ? 1 : 0], st));
  net->bwd_next_stage = stage - 1;
  if (stage == 0) net->bwd_blocks = false;
  return DIRB200_OK;
}

/* Parameters of stage `stage` (0 = stem conv1 + bn1, s = layer group s) occupy [*lo, *hi) of the flat buffers. */
int dirb200_resnet_stage_param_range(const dirb200_net* net, int stage, int64_t* lo, int64_t* hi) {
  DIRB_CHECK_ARG(net && lo && hi, "resnet_stage_param_range: null pointer");
  const int nst = (int)net->stage_begin.size() - 2;
  DIRB_CHECK_ARG(stage >= 0 && stage <= nst, "resnet_stage_param_range: bad stage %d", stage);
  auto first = [&](int s) -> int64_t {
    return s > nst ? (int64_t)net->param_count : (int64_t)net->blocks[net->stage_begin[s]].c1.w_off;
  };
  *lo = stage == 0 ? 0 : first(stage);
  *hi = first(stage + 1);
  return DIRB200_OK;
}

int dirb200_resnet_num_stages(const dirb200_net* net) { return net ? (int)net->stage_begin.size() - 2 : -1; }

/* d_enc fp32 [n, feature_dim] -> ACCUMULATES d loss / d parameter into grads (flat fp32, same layout as params): all
 * stages back to back.  Must follow a training-mode forward on the same net. */
int dirb200_resnet_backward(dirb200_net* net, const float* d_enc, const float* params, float* grads, void* stream) {
  DIRB_CHECK_ARG(net && d_enc && params && grads, "resnet_backward: null pointer");
  for (int stage = (int)net->stage_begin.size() - 2; stage >= 0; --stage)
    RUN(dirb200_resnet_backward_stage(net, stage, d_enc, params, grads, stream));
  return DIRB200_OK;
}

}  // extern "C"

extern "C" {
/* Test / debugging aid: device pointer and shape of an internal activation.
 * block = -1: stem (which 0 = conv1 raw, 1 = relu(bn1), 6 = max-pool output, 7 = max-pool argmax);
 * block >= 0: which 0/1 = conv1 raw / act, 2/3 = conv2 raw / act, 4 = conv3 raw, 5 = downsample raw, 6 = block output,
 * 7 = the block output's ReLU mask.  Selectors 7 report bytes: *channels is the row length in bytes. */
int dirb200_resnet_peek(dirb200_net* net, int block, int which, void** ptr, int64_t* rows, int* channels) {
  // the selector is checked before the net is dereferenced
  DIRB_CHECK_ARG(which >= 0 && which <= 7, "resnet_peek: bad selector %d", which);
  DIRB_CHECK_ARG(block != -1 || which <= 1 || which >= 6, "resnet_peek: bad selector %d for the stem", which);
  DIRB_CHECK_ARG(net && ptr && rows && channels, "resnet_peek: null pointer");
  DIRB_CHECK_ARG(block >= -1 && block < (int)net->blocks.size(), "resnet_peek: bad block %d", block);
  const ConvLayer* cv = nullptr;
  bool act = false;
  if (which == 7 && block >= 0) {
    // only a training-mode forward writes the masks (the backward pass reads them); after any other they are stale
    DIRB_CHECK_ARG(net->forward_was_training,
                   "resnet_peek: block ReLU mask not materialised (written by a training-mode forward only)");
    const Block& B = net->blocks[block];
    *ptr = B.mask; *rows = B.c3.rows; *channels = B.c3.s.cout / 8;
    return DIRB200_OK;
  }
  if (block < 0) {
    const int64_t pool_rows = (int64_t)net->n * net->pool_h * net->pool_w;
    if (which == 6 || which == 7) {
      *ptr = which == 6 ? (void*)net->pool_out : (void*)net->pool_idx; *rows = pool_rows; *channels = 64;
      return DIRB200_OK;
    }
    cv = &net->stem; act = which == 1;
  } else {
    Block& B = net->blocks[block];
    switch (which) {
      case 0: cv = &B.c1; break;
      case 1: cv = &B.c1; act = true; break;
      case 2: cv = &B.c2; break;
      case 3: cv = &B.c2; act = true; break;
      case 4: cv = &B.c3; break;
      case 5: DIRB_CHECK_ARG(B.has_ds, "resnet_peek: block has no downsample"); cv = &B.ds; break;
      case 6: *ptr = B.out; *rows = B.c3.rows; *channels = B.c3.s.cout; return DIRB200_OK;
      default: DIRB_CHECK_ARG(false, "resnet_peek: bad selector %d", which);
    }
  }
  *ptr = act ? cv->a : cv->y;
  *rows = cv->rows;
  *channels = cv->s.cout;
  DIRB_CHECK_ARG(*ptr, "resnet_peek: tensor not materialised");
  return DIRB200_OK;
}

/* Test / debugging aid: one conv layer's buffers, offset, shape and the split factor of its reduction-table entry.
 * block = -1: stem (conv 0); block >= 0: conv 0 / 1 / 2 / 3 = conv1 / conv2 / conv3 / downsample. */
// The conv layer (block, conv) names and its entry in the split-K reduction table; `who` prefixes the refusals.
static int find_conv(const dirb200_net* net, int block, int conv, const char* who, const ConvLayer** cv_out,
                     int* entry_out) {
  DIRB_CHECK_ARG(block >= -1 && block < (int)net->blocks.size(), "%s: bad block %d", who, block);
  DIRB_CHECK_ARG(conv >= 0 && conv <= (block < 0 ? 0 : 3), "%s: bad conv %d", who, conv);
  // the reduction table holds the stem, then every block's c1, c2, c3 [, ds] in block order (build())
  int entry = 0;
  const ConvLayer* cv = &net->stem;
  if (block >= 0) {
    const Block& B = net->blocks[block];
    DIRB_CHECK_ARG(conv < 3 || B.has_ds, "%s: block %d has no downsample", who, block);
    entry = 1;
    for (int b = 0; b < block; ++b) entry += net->blocks[b].has_ds ? 4 : 3;
    entry += conv;
    const ConvLayer* convs[4] = {&B.c1, &B.c2, &B.c3, &B.ds};
    cv = convs[conv];
  }
  *cv_out = cv;
  *entry_out = entry;
  return DIRB200_OK;
}

int dirb200_resnet_peek_conv(dirb200_net* net, int block, int conv, dirb200_conv_peek* out) {
  DIRB_CHECK_ARG(net && out, "resnet_peek_conv: null pointer");
  int entry = 0;
  const ConvLayer* cv = nullptr;
  RUN(find_conv(net, block, conv, "resnet_peek_conv", &cv, &entry));
  WgradReduceDesc d{};
  DIRB_CUDA(cudaMemcpy(&d, net->reduce_descs + entry, sizeof(d), cudaMemcpyDeviceToHost));
  DIRB_CHECK_ARG(d.partial == cv->wpart && d.w_off == cv->w_off,
                 "resnet_peek_conv: reduction-table entry %d does not belong to this conv", entry);
  out->w_fprop = cv->wf;
  out->w_dgrad = cv->wd;
  out->partial = cv->wpart;
  out->scale = cv->bn.scale;
  out->shift = cv->bn.shift;
  out->w_off = (int64_t)cv->w_off;
  if (cv->stem) {
    out->cout = cv->s.cout; out->cin = 3; out->kh = 7; out->kw = 7; out->stride = 2; out->pad = 3;
  } else {
    out->cout = cv->s.cout; out->cin = cv->s.cin; out->kh = cv->s.kh; out->kw = cv->s.kw; out->stride = cv->s.stride;
    out->pad = cv->s.pad;
  }
  out->stem = cv->stem ? 1 : 0;
  out->splits = d.splits;
  return DIRB200_OK;
}

/* Test / debugging aid: one conv's BatchNorm batch statistics (fp32 [cout] mean, invstd) of the last training-mode
 * forward.  block / conv as dirb200_resnet_peek_conv. */
int dirb200_resnet_peek_bn_stats(dirb200_net* net, int block, int conv, float** mean, float** invstd) {
  DIRB_CHECK_ARG(net && mean && invstd, "resnet_peek_bn_stats: null pointer");
  int entry = 0;
  const ConvLayer* cv = nullptr;
  RUN(find_conv(net, block, conv, "resnet_peek_bn_stats", &cv, &entry));
  *mean = cv->bn.mean;
  *invstd = cv->bn.invstd;
  return DIRB200_OK;
}
}
