/* dirb200.h -- C ABI of libdirb200.so: the H100-native (sm_90a) hot path of
 * YyzHarry/imbalanced-regression (ResNet-50 + FDS + LDS training step).
 *
 * The reference has no FFI: its "plugin boundary" for this path is a set of
 * Python callables (SURVEY.md §8b).  Each entry point below names the
 * reference function it replaces (file:line in the reference repository); the
 * Python host mirrors in imbalanced-regression_b200/{fds,loss,utils,resnet,
 * datasets}.py keep the reference's names/signatures and call these through
 * ctypes (see INTEGRATION.md).
 *
 * Conventions
 *  - plain C types only; every pointer is a DEVICE pointer unless the name
 *    ends in _host; the caller owns all memory, nothing is allocated here
 *    except inside the opaque dirb200_net object;
 *  - every function returns 0 on success, <0 on error (message via
 *    dirb200_last_error(), thread local); nothing throws, nothing
 *    synchronises the host, every launch goes to the cudaStream_t passed
 *    (as void*; NULL = legacy default stream);
 *  - there is NO CPU fallback: without a CUDA device every compute entry
 *    point fails with DIRB200_ERR_CUDA.
 */
#ifndef DIRB200_H
#define DIRB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DIRB200_OK 0
#define DIRB200_ERR_ARG (-1)
#define DIRB200_ERR_CUDA (-2)
#define DIRB200_ERR_WORKSPACE (-3)

/* bin rules (row label -> FDS table row) */
#define DIRB200_BIN_AGE 0     /* agedb-dir/fds.py:91-99 : int(label - bucket_start), edge folding */
#define DIRB200_BIN_DEPTH10 1 /* nyud2-dir/models/fds.py:51-53 : clamp(int(label*10), bucket_start, bucket_num-1) */
#define DIRB200_BIN_EDGES5 2  /* sts-b-dir/fds.py:51-57 : np.histogram edges over [0,5], bucket_num bins */
/* the rule also selects calibrate_mean_var's channel mask: v1 != 0 (age, agedb-dir/utils.py:100) or
 * v1 > 0 && v2 >= 0 (nyud2-dir/util.py:154, sts-b-dir/util.py:66) */

/* loss kinds (agedb-dir/loss.py) */
#define DIRB200_LOSS_MSE 0       /* loss.py:5-10  */
#define DIRB200_LOSS_L1 1        /* loss.py:13-18 */
#define DIRB200_LOSS_FOCAL_MSE 2 /* loss.py:21-28 */
#define DIRB200_LOSS_FOCAL_L1 3  /* loss.py:31-38 */
#define DIRB200_LOSS_HUBER 4     /* loss.py:41-48 */
#define DIRB200_ACT_SIGMOID 0
#define DIRB200_ACT_TANH 1

/* LDS re-weighting (agedb-dir/datasets.py:64-67) */
#define DIRB200_REWEIGHT_SQRT_INV 1
#define DIRB200_REWEIGHT_INVERSE 2

const char* dirb200_last_error(void);
int dirb200_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t dirb200_launch_count(void);

/* ---------------------------------------------------------------- FDS ---- */

/* Edge-label presence flags: flags[0] |= any(label == bucket_start),
 * flags[1] |= any(label == bucket_num-1).  The caller zeroes flags (int32[2])
 * and may OR-reduce them across ranks.  Replaces the `label == bucket_start`
 * / `label == bucket_num-1` branches of the unique-label loop,
 * agedb-dir/fds.py:94-97,124-137. */
int dirb200_fds_label_flags(const float* labels, int64_t n, int bucket_num, int bucket_start,
                            int bin_rule, int32_t* flags, void* stream);

/* Row -> table row (int32, -1 = untouched), agedb-dir/fds.py:91-99. */
int dirb200_fds_bin_rows(const float* labels, int64_t n, int bucket_num, int bucket_start,
                         int bin_rule, const int32_t* flags, int32_t* bins_out, void* stream);

/* Workspace for dirb200_fds_accumulate. */
size_t dirb200_fds_accumulate_workspace_bytes(int64_t n, int nb);

/* Segmented (per label bin) accumulation of sum / sum-of-squares in fp64 and
 * row counts over features[n,d] (fp32 row-major, each element read exactly
 * once).  ADDS into sums/sumsq [nb,d] (double) and counts [nb] (int64), so an
 * epoch can be streamed batch by batch with no host round trip; the caller
 * zeroes them at epoch start and may all-reduce(sum) them across ranks.
 * Replaces the per-label mask/gather/mean/var loop, agedb-dir/fds.py:91-102,
 * and the host round trip at agedb-dir/train.py:276-279. */
int dirb200_fds_accumulate(const float* features, const int32_t* bins, int64_t n, int d, int nb,
                           double* sums, double* sumsq, int64_t* counts,
                           void* workspace, size_t workspace_bytes, void* stream);

/* Measurement aid (bench.py's `roofline` line; no reference counterpart): when enabled, dirb200_fds_accumulate
 * records CUDA events on the caller's stream around its fds_accumulate_kernel launch alone (the counting sort
 * that precedes it is excluded); dirb200_fds_last_accumulate_kernel_ms synchronises on them and returns the
 * kernel's duration of the most recent call. */
int dirb200_fds_set_profiling(int enabled);
int dirb200_fds_last_accumulate_kernel_ms(float* ms_out);

/* mean/var (unbiased; 0 when n==1) from the accumulators, then the running
 * EMA update of every bin with count>0, agedb-dir/fds.py:100-111.
 * momentum < 0 selects the `momentum is None` rule (factor = 1 - n/tracked);
 * first_update != 0 forces factor 0 (epoch == start_update, fds.py:107). */
int dirb200_fds_finalize(const double* sums, const double* sumsq, const int64_t* counts, int nb, int d,
                         float* running_mean, float* running_var, float* num_samples_tracked,
                         double momentum, int first_update, void* stream);

/* dst[b,:] = sum_j window[j] * src[reflect(b + j - (ks-1)/2), :]; ks <= 33.
 * Replaces F.pad(reflect)+F.conv1d, agedb-dir/fds.py:58-67. */
int dirb200_fds_smooth_tables(const float* src, int nb, int d, const float* window_host, int ks,
                              float* dst, void* stream);

/* In-place whiten/re-colour of x[b,d] by label bin: FDS.smooth +
 * calibrate_mean_var (agedb-dir/fds.py:115-144, agedb-dir/utils.py:97-107).
 * Edge flags are evaluated on this batch's labels (as the reference does per
 * call).  rowbin_out[b] (int32) = table row used, or -1 when the row was left
 * untouched (label dropped, or sum(v1[row]) < 1e-10): the backward's input. */
int dirb200_fds_calibrate_fwd(float* x, const float* labels, int64_t b, int d, int bucket_num,
                              int bucket_start, int bin_rule, const float* m1, const float* v1,
                              const float* m2, const float* v2, float clip_min, float clip_max,
                              int32_t* rowbin_out, int32_t* flags_scratch /* int32[2]; may be NULL when b <= 2048 */,
                              void* stream);

/* STS-B variant (sts-b-dir/fds.py:112-125): buckets with counts[b] == 0 in this update take their neighbours'
 * running statistics (copy at the two ends, mean of both neighbours inside), in increasing bucket order. */
int dirb200_fds_fill_empty(const int64_t* counts, int nb, int d, float* running_mean, float* running_var,
                           void* stream);

/* grad_in[b,d] = grad_out[b,d] * d(calibrate)/dx (may alias). */
int dirb200_fds_calibrate_bwd(int bin_rule, const float* grad_out, const int32_t* rowbin, int64_t b, int d,
                              const float* v1, const float* v2, float clip_min, float clip_max,
                              float* grad_in, void* stream);

/* ------------------------------------------------------------- losses ---- */

size_t dirb200_loss_workspace_bytes(int64_t n);

/* Fused forward + backward of weighted_{mse,l1,focal_mse,focal_l1,huber}_loss
 * (agedb-dir/loss.py:5-48): loss_out[0] = mean(l_i * w_i); if grad_out != NULL,
 * grad_out[i] = grad_scale * d loss / d pred_i.  weight may be NULL. */
int dirb200_loss_fwd_bwd(int kind, const float* pred, const float* target, const float* weight, int64_t n,
                         float beta, float gamma, int activate, float grad_scale,
                         float* loss_out, float* grad_out, void* workspace, size_t workspace_bytes,
                         void* stream);

/* ---------------------------------------------------------------- LDS ---- */

/* hist[min(max_target-1, int(label))]++ (int64, bit exact), ADDS into hist so
 * it can be all-reduced when labels are sharded.  agedb-dir/datasets.py:60-63. */
int dirb200_lds_histogram(const float* labels, int64_t n, int max_target, int64_t* hist, void* stream);

/* hist -> per-bin value (sqrt / clip(5,1000), optional convolve1d(mode=constant)
 * with the float64 window, integer truncation on the 'inverse' path as scipy
 * does) -> per-sample float32 weight 1/value[bin] scaled to mean 1.
 * scratch: >= (2*max_target + 2) doubles.  agedb-dir/datasets.py:64-82. */
int dirb200_lds_weights(const float* labels, int64_t n, int max_target, int reweight,
                        const double* window_host, int ks, const int64_t* hist,
                        double* scratch, float* weights_out, void* stream);

/* Same, for a label column sharded over ranks: `hist` is the histogram of the WHOLE column (the per-rank
 * dirb200_lds_histogram outputs SUM-all-reduced, int64, exact) and `n_total` its length; the per-bin table and the
 * len / sum(w) normaliser (agedb-dir/datasets.py:81-82) are formed from those, the gather covers this rank's
 * `n` labels.  dirb200_lds_weights == this with n_total = n.  SURVEY.md section 8e(3). */
int dirb200_lds_weights_sharded(const float* labels, int64_t n, int64_t n_total, int max_target, int reweight,
                                const double* window_host, int ks, const int64_t* hist, double* scratch,
                                float* weights_out, void* stream);

/* Dense per-element weight lookup of nyud2-dir/loaddata.py:52-64: weights_out[i] = table[min(int(values[i] * mult),
 * max_bin)] (mult = 10, max_bin = 99 for depth maps; table = the bucket weights, device pointer). */
int dirb200_lds_table_lookup(const float* values, int64_t n, float mult, int max_bin, const float* table,
                             float* weights_out, void* stream);

/* ------------------------------------------------ BatchNorm / pooling layers ---- */
/* nn.BatchNorm2d in training mode on an NHWC bf16 tensor y [rows][c] (rows = N*H*W > 0; c = 8, 16, 32, ..., 2048:
 * c / 8 channel groups must divide a CTA's 256 threads, so e.g. c = 24 is refused),
 * optionally followed by ReLU (agedb-dir/resnet.py:46-51,128-130; nyud2-dir/models/modules.py:13-21): batch statistics
 * (biased variance) -> running statistics updated in place with `momentum` (unbiased variance; NULL: not tracked) ->
 * out = [relu](gamma * (y - mean) * invstd + beta).  save_mean / save_invstd [c] and scale_shift [2][c] are kept for
 * the backward.  workspace: dirb200_bn_workspace_bytes(c). */
size_t dirb200_bn_workspace_bytes(int c);
int dirb200_bn_train_fwd(const void* y, int64_t rows, int c, const float* gamma, const float* beta, float eps,
                         float momentum, float* running_mean, float* running_var, int relu, void* out, float* save_mean,
                         float* save_invstd, float* scale_shift, void* workspace, void* stream);
/* Eval mode (nn.BatchNorm2d under model.eval()): scale = gamma * rsqrt(running_var + eps), shift = beta -
 * running_mean * scale (fp32 [c]); the running statistics are only read.  dirb200_layer_bn_apply applies them. */
int dirb200_bn_eval_coeffs(int c, const float* gamma, const float* beta, float eps, const float* running_mean,
                           const float* running_var, float* scale, float* shift, void* stream);
/* grad_out = d loss / d out -> grad_y = d loss / d y (bf16), grad_gamma / grad_beta ACCUMULATED (fp32 [c]).  With relu the
 * mask is re-derived from (y, scale_shift) -- the activation itself is not read. */
int dirb200_bn_train_bwd(const void* grad_out, const void* y, int64_t rows, int c, const float* gamma,
                         const float* save_mean, const float* save_invstd, const float* scale_shift, int relu,
                         float* grad_gamma, float* grad_beta, void* grad_y, void* workspace, void* stream);
/* nn.MaxPool2d(kernel_size=3, stride=2, padding=1) (resnet.py:82) on NHWC bf16, argmax (r*3+s of the first maximum)
 * kept as one byte per output element; backward for even H, W. */
int dirb200_maxpool3x3s2_fwd(const void* x, int n, int h, int w, int c, void* out, uint8_t* argmax, void* stream);
int dirb200_maxpool3x3s2_bwd(const void* grad_out, const uint8_t* argmax, int n, int h, int w, int c, void* grad_x,
                             void* stream);
/* nn.AvgPool2d over the whole hw-pixel map (resnet.py:87) : NHWC bf16 [n][hw][c] <-> fp32 [n][c] */
int dirb200_avgpool_fwd(const void* x, int n, int hw, int c, float* out, void* stream);
int dirb200_avgpool_bwd(const float* grad_out, int n, int hw, int c, void* grad_x, void* stream);

/* ------------------------------------------------ dense-prediction ops (NYUD2-DIR) ---- */
/* The NYUD2 decoder / feature-fusion / refinement modules (nyud2-dir/models/modules.py:6-174) are 1x1 / 3x3 / 5x5
 * convolutions (dirb200_conv_fprop / _dgrad / _wgrad take filters up to 5x5 at stride 1), bilinear up-sampling and a
 * channel concat.  NHWC bf16 like the conv stage; channel counts multiples of 8.
 * upsample: F.upsample(x, size=(ho, wo), mode='bilinear') with align_corners = False (modules.py:24), the weights
 * formed and associated as ATen does; the backward is a deterministic gather (ATen scatters with atomics). */
int dirb200_upsample_bilinear_fwd(const void* x, int n, int h, int w, int c, int ho, int wo, void* out, void* stream);
int dirb200_upsample_bilinear_bwd(const void* dy, int n, int h, int w, int c, int ho, int wo, void* dx, void* stream);
/* dst[p][dst_off + j] = src[p][src_off + j] for j < c, p < pixels (row strides in elements): torch.cat(..., 1) of
 * NHWC tensors (modules.py:120) is one call per source; its backward is the same call with the roles swapped. */
int dirb200_copy_channels(const void* src, int src_stride, int src_off, void* dst, int dst_stride, int dst_off, int c,
                          int64_t pixels, void* stream);
/* The depth head of module R (modules.py:145, 169: conv2 = nn.Conv2d(c, 1, kernel_size=5, stride=1, padding=2,
 * bias=True), x2 = conv2(x1_s)) as memory-bound kernels written for one output channel.  x bf16 NHWC [n, h, w, c];
 * w fp32 [1, c, 5, 5] and b fp32 [1], the reference's parameters as they are.  c a multiple of 8 from 8 to 256,
 * n, h, w > 0, n * h * w * c < 2^31.  Deterministic: every sum has a fixed order (no atomics), so repeated calls give
 * the same bits and one image's output does not depend on the rest of the batch.
 * fwd:   y fp32 [n, h, w, 1] (the bytes of the reference's [n, 1, h, w]) = b + sum_{ch, tap} w * x, fp32 accumulation.
 * dgrad: dx bf16 [n, h, w, c], dx[p, ch] = sum_tap w[ch, tap] * dy[p - tap], one rounding of an fp32 sum; dy fp32.
 * wgrad: dw fp32 [1, c, 5, 5], dw[ch, tap] = sum_p dy[p] * x[p + tap, ch], and db fp32 [1] = sum_p dy[p], both
 *        overwritten; per-tile partials in the workspace, reduced in tile order. */
int dirb200_depth_head_fwd(const void* x, const float* w, const float* b, float* y, int n, int h, int wd, int c,
                           void* stream);
int dirb200_depth_head_dgrad(const float* dy, const float* w, void* dx, int n, int h, int wd, int c, void* stream);
size_t dirb200_depth_head_wgrad_workspace_bytes(int n, int h, int wd, int c);     /* 0 for a refused shape */
int dirb200_depth_head_wgrad(const void* x, const float* dy, float* dw, float* db, void* workspace,
                             size_t workspace_bytes, int n, int h, int wd, int c, void* stream);

/* ------------------------------------------------ input pipeline ---- */
/* Batched device form of the per-sample torchvision chain agedb-dir/datasets.py:38-53 after the resize:
 * RandomCrop(size, padding=pad) -> RandomHorizontalFlip -> ToTensor -> Normalize(mean, std), bit-identical to
 * torchvision for the same draws.  images u8 [n][size][size][3] (RGB, HWC) -> out f32 [n][3][size][size].
 * crop_yx int32 [n][2] = (top, left) of the crop in the zero-padded image, 0 .. 2*pad (NULL: (pad, pad) = the
 * validation chain, :46-51); flip u8 [n] (NULL: no flips).  value = (u8 / 255 - mean) / std; padding = u8 0. */
int dirb200_augment_batch(const uint8_t* images, const int* crop_yx, const uint8_t* flip, int n, int size, int pad,
                          float mean, float stdv, float* out, void* stream);

/* Batched device form of NYUD2-DIR's per-sample chains after Scale(240) (nyud2-dir/loaddata.py:108-125 training,
 * :132-148 FDS, :151-170 test, with nyud2-dir/nyu_transform.py), plus _get_weights (loaddata.py:58-67).
 * images u8 [n][h][w][3] (RGB, HWC); depths u8 [n][h][w] (depth_u16 = 0) or u16 [n][h][w] (depth_u16 = 1: the test
 * chain, int16 / 1000, no flip / rotation / resize).  Outputs: image_out f32 [n][3][crop_h][crop_w], depth_out and
 * weight_out f32 [n][1][depth_h][depth_w] (weight_out may be NULL without a table).
 *   flip u8 [n] (NULL: none): RandomHorizontalFlip, before the rotation (nyu_transform.py:55-71);
 *   affine f64 [n][6] = (m00, m01, m10, m11, offset0, offset1) of scipy.ndimage.rotate(reshape=False) over the
 *     (h, w) plane (NULL: no rotation): RandomRotate(5), order-2 spline, mode 'constant' (:24-53), bit-exact uint8;
 *   CenterCrop at (round((w - crop_w) / 2), round((h - crop_h) / 2)), half to even; the depth crop resized to
 *     depth_h x depth_w by Pillow's 8-bit BICUBIC (:118-148), bit-exact; ToTensor: u8 / 255, depth * 10 (:151-213);
 *   rgb_offset f32 [n][3] (NULL: none): Lighting's per-channel offset (:216-236), computed on the host;
 *   jitter_order i32 [n][3] (0 brightness, 1 contrast, 2 saturation) and jitter_alpha f32 [n][3], the weight of the
 *     k-th applied transform (NULL, NULL: none): ColorJitter (:239-312); Contrast's mean is reduced in fp64;
 *   mean_std: HOST f32 [6], Normalize's mean then std (:315-347);
 *   bucket_weights f32 [n_buckets >= 100] on the device: weight = table[min(int(depth * 10), 99)] (NULL: ones).
 * debug_crop u8 [n][crop_h][crop_w][4] (R, G, B, depth after flip + rotation + crop) and debug_mean f32 [n] (Contrast's
 * grayscale mean; written only with jitter): optional test outputs, NULL to skip.
 * Every argument is checked before any CUDA call. */
size_t dirb200_depth_augment_workspace_bytes(int n, int h, int w, int crop_h, int crop_w);
int dirb200_depth_augment_batch(const uint8_t* images, const void* depths, int depth_u16, int n, int h, int w,
                                int crop_h, int crop_w, int depth_h, int depth_w, const uint8_t* flip,
                                const double* affine, const float* rgb_offset, const int* jitter_order,
                                const float* jitter_alpha, const float* mean_std, const float* bucket_weights,
                                int n_buckets, float* image_out, float* depth_out, float* weight_out,
                                uint8_t* debug_crop, float* debug_mean, void* workspace, size_t workspace_bytes,
                                void* stream);

/* ------------------------------------------------ evaluation metrics ---- */
/* hist[int(label)] += 1 for 0 <= int(label) < nbins (int64, bit-exact, ADDS; no clamping): the per-label-value
 * training counts that shot_metrics compares against, agedb-dir/train.py:339,350. */
int dirb200_int_label_histogram(const float* labels, int64_t n, int nbins, int64_t* hist, void* stream);

/* Overall and many / median / low-shot error sums of a prediction vector in one pass (replaces the host loop over
 * np.unique(labels) of shot_metrics, agedb-dir/train.py:338-391, and the MSE / L1 / G-Mean meters of validate,
 * :286-335).  A sample is "many"-shot when the training count of its label value is > many_shot_thr, "low" when
 * it is < low_shot_thr (label values absent from training or not integer valued count 0), else "median".
 * out16 (double[4][4], OVERWRITTEN): rows = overall, many, median, low; columns = count, sum (pred-label)^2,
 * sum |pred-label|, sum log|pred-label|  ->  mse = c1/c0, l1 = c2/c0, gmean = exp(c3/c0). */
int dirb200_shot_metrics(const float* preds, const float* labels, int64_t n, const int64_t* train_hist, int nbins,
                         int many_shot_thr, int low_shot_thr, double* out16, void* stream);

/* NYUD2-DIR depth evaluation in one fused pass (replaces nyud2-dir/test.py:52-55 -- F.interpolate(align_corners=True),
 * output[mask], the per-image .cpu() -- and Evaluator.__call__ / evaluate / evaluate_shot, nyud2-dir/util.py:35-133).
 * pred fp32 [n_images][ph][pw]; target fp32 and mask u8 [n_images][h][w] (mask NULL: every pixel).  When
 * (ph, pw) != (h, w) the prediction is ATen's CUDA upsample_bilinear2d with align_corners = True, formed in registers
 * for the masked pixels only; equal sizes copy.  Per-pixel terms in fp32 as Evaluator.evaluate forms them (a NaN
 * target zeroes them), widened to fp64 and summed.  Shot group of a finite target: bin = min(int(t * 10.f), 99)
 * (fp32 product, truncation toward zero), group_of_bin[bin] for 0 <= bin < nbins (u8: 0 none, 1 many, 2 medium,
 * 3 few; NULL iff nbins == 0); NaN / inf targets belong to no group.
 * acc double[4][10], ADDED to (stream an evaluation batch by batch): rows overall, many, medium, few; columns NUM
 * (non-NaN targets), sum d^2, sum d, sum d/t, sum |lg10 o - lg10 t|, delta1-3 counts (max(o/t, t/o) <= 1.25^k),
 * NaN-target count, +-inf-target count (d = |o - t|).  Deterministic: per-CTA partials in `workspace`, summed in
 * CTA order by the last CTA; one kernel launch. */
size_t dirb200_depth_metrics_workspace_bytes(int64_t n_images, int h, int w);
int dirb200_depth_metrics_accumulate(const float* pred, int ph, int pw, const float* target, const uint8_t* mask,
                                     int64_t n_images, int h, int w, const uint8_t* group_of_bin, int nbins,
                                     double* acc, void* workspace, size_t workspace_bytes, void* stream);

/* STS-B-DIR's STSShotAverage.get_metric (replaces sts-b-dir/util.py:123-172, metrics mse / l1 / gmean / pearsonr /
 * spearmanr as tasks.py:86 asks for them) over n fp32 predictions and labels (n <= 2^22):
 * out24[g * 6 + k], g = 0 overall, 1 many, 2 medium, 3 few; k = 0 num_samples, 1 MSE, 2 L1, 3 G-mean, 4 Pearson,
 * 5 Spearman, all fp64 with x = 5 pred.  A label's group is its DIRB200_BIN_EDGES5 bin over 50 bins in util.py:110-113's
 * table (a negative label: few).  An exact zero difference enters the G-mean as 1e-10; Pearson is scipy's centred
 * formula clipped to [-1, 1] (rounded at n = 2, NaN for a constant input); Spearman is the Pearson of the average ranks
 * within the group, found exactly by an O(n^2) pair count; a group of size 0 reports 0 everywhere, one of size 1 0 for
 * both correlations.  Two launches, no floating-point atomics: identical calls give identical bits.  workspace: 16 n
 * bytes, 16-byte aligned (none for n = 0). */
size_t dirb200_stsb_shot_metrics_workspace_bytes(int64_t n);
int dirb200_stsb_shot_metrics(const float* preds, const float* labels, int64_t n, void* workspace,
                              size_t workspace_bytes, double* out24, void* stream);

/* ------------------------------------------------- convolution stack ---- */
/* Activations are NHWC bf16; weights arrive in the reference's fp32
 * [Cout][Cin][KH][KW] layout (agedb-dir/resnet.py:46-51,79,112-118, i.e. the
 * nn.Conv2d parameters / state_dict tensors) and are re-laid-out to bf16 GEMM
 * operands by dirb200_conv_prep_weights.  The convolutions themselves are
 * wgmma implicit GEMMs (fp32 accumulate in registers); they replace the cuDNN
 * calls behind nn.Conv2d forward and its autograd backward.
 * Cin and Cout must be multiples of 64, except the stem (stem=1: Cin=3, 7x7,
 * stride 2, pad 3), which consumes the 16-channel space-to-depth input made
 * by dirb200_input_to_s2d. */

/* w fp32 [Cout][Cin][KH][KW] -> w_fprop bf16 [Cout][KH][KW][Cin] and (if not
 * NULL) w_dgrad bf16 [Cin][KH][KW][Cout].  stem: w_fprop bf16 [Cout][256]. */
int dirb200_conv_prep_weights(const float* w, int cout, int cin, int kh, int kw, int stem,
                              void* w_fprop, void* w_dgrad, void* stream);

/* x fp32 NCHW [n,3,h,w] (what ResNet.forward receives, resnet.py:127) ->
 * bf16 [n, h/2, w/2, 16], channel (ph*2+pw)*4+c, c==3 zero. */
int dirb200_input_to_s2d(const float* x_nchw, int n, int h, int w, void* out_bf16, void* stream);

/* y[n,ho,wo,cout] = conv2d(x[n,h,w,cin], w)  (bias-free, as every conv in resnet.py) */
int dirb200_conv_fprop(const void* x, const void* w_fprop, void* y, int n, int h, int w, int cin,
                       int cout, int kh, int kw, int stride, int pad, int stem, void* stream);

/* dx[n,h,w,cin] = d loss / d x given dy[n,ho,wo,cout] */
int dirb200_conv_dgrad(const void* dy, const void* w_dgrad, void* dx, int n, int h, int w, int cin,
                       int cout, int kh, int kw, int stride, int pad, void* stream);

/* Host-only (no CUDA call, works without a device): which GEMM form the three entry points above / below would launch for
 * a shape (op: 0 fprop, 1 dgrad, 2 wgrad).  plan7[0] tile width BN; [1] 0 (no CTA pairs on
 * sm_90a); [2] A-operand form: 0 cp.async gather, 1 tiled TMA, 2 im2col-mode TMA; [3] 0 (no patch-resident form on
 * sm_90a); [4] split-K factor (wgrad); [5] launches (a stride-2
 * dgrad runs one per non-empty output-pixel parity class); [6] 1 = this dgrad can also accumulate the BN-backward
 * moments of the previous layer in its epilogue. */
int dirb200_conv_plan(int n, int h, int w, int cin, int cout, int kh, int kw, int stride, int pad, int stem, int op,
                      int* plan7);
size_t dirb200_conv_wgrad_workspace_bytes(int n, int h, int w, int cin, int cout, int kh, int kw,
                                          int stride, int pad, int stem);

/* dw fp32 [Cout][Cin][KH][KW] (=, or += when accumulate) d loss / d w from x and dy
 * (split-K partials in `workspace`, then a deterministic reduce). */
int dirb200_conv_wgrad(const void* x, const void* dy, float* dw, void* workspace, size_t workspace_bytes,
                       int n, int h, int w, int cin, int cout, int kh, int kw, int stride, int pad,
                       int stem, int accumulate, void* stream);

/* ------------------------------------------------ Test aids: fused conv epilogues ---- */
/* The network runner fuses BatchNorm work into the conv epilogues; these entry points run one such launch alone so
 * that it can be checked against a high-precision reference.  A statistics row layout crosses the ABI as a host
 * int[4] {rows, n_tiles, bn, group}: channel ch is held in rows (j + k*n_tiles)*group + r, j = ch / bn, k = 0, 1, ..
 * while the row index < rows, r < group.  Every row the layout names for a channel is written, nothing else.
 * partial: fp32 [rows][2][C], at most (max(SMs, C / 64) x 2 x C) floats, C = cout (fprop) or cin (dgrad); rows is
 * min(tiles, SMs), raised to the C / bn column tiles where the SM count is capped below that (DIRB200_SMS). */

/* dirb200_conv_fprop that also writes the per-channel sum (slot 0) and sum of squares (slot 1) of the stored bf16 y. */
int dirb200_conv_fprop_bn_stats(const void* x, const void* w_fprop, void* y, int n, int h, int w, int cin, int cout,
                                int kh, int kw, int stride, int pad, int stem, float* partial, int* layout_host,
                                void* stream);
/* Inference form (BatchNorm folded into the conv): out = [relu](conv(x, w) * scale[co] + shift[co]) without a
 * residual; with one (NULL: none; [pixels][cout] bf16) out = [relu](bf16(conv * scale + shift) + residual). */
int dirb200_conv_fprop_affine(const void* x, const void* w_fprop, void* out, int n, int h, int w, int cin, int cout,
                              int kh, int kw, int stride, int pad, const float* scale, const float* shift,
                              const void* residual, int relu, void* stream);
/* dirb200_conv_dgrad (stride 1; dirb200_conv_plan's plan7[6] says where it applies) that also writes the backward
 * moments of the BatchNorm + ReLU before it: dz = dx_stored * [y_prev * scale + shift > 0], slot 0 = sum dz,
 * slot 1 = sum dz * y_prev.  y_prev: [pixels][cin] bf16 like dx. */
int dirb200_conv_dgrad_bn_moments(const void* dy, const void* w_dgrad, void* dx, int n, int h, int w, int cin, int cout,
                                  int kh, int kw, int stride, int pad, const void* y_prev, const float* scale,
                                  const float* shift, float* partial, int* layout_host, void* stream);
/* BatchNorm batch statistics from the rows of dirb200_conv_fprop_bn_stats (rows = pixels): mean, invstd (biased
 * variance), scale = gamma * invstd, shift = beta - mean * scale; running statistics (NULL: not tracked) updated with
 * `momentum` and the unbiased variance. */
int dirb200_bn_finalize_layout(const float* partial, const int* layout_host, int64_t rows, int c, const float* gamma,
                               const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                               float* mean_out, float* invstd_out, float* scale_out, float* shift_out, void* stream);
/* BatchNorm backward coefficients from the rows of dirb200_conv_dgrad_bn_moments: dgamma = invstd * (S1 - mean * S0),
 * dbeta = S0 (both ACCUMULATED into grad_gamma / grad_beta); coef_out [3][c] = A, B, C of dy = A*dz + B*y + C. */
int dirb200_bn_bwd_coeffs_layout(const float* partial, const int* layout_host, int64_t rows, int c, const float* mean,
                                 const float* invstd, const float* gamma, float* grad_gamma, float* grad_beta,
                                 float* coef_out, void* stream);

/* ------------------------------------------------ Test aids: BatchNorm / pooling layer kernels ---- */
/* The HBM-bound layer kernels the runner and the BatchNorm entry points above sequence, one launch per call with the
 * runner's own dispatch, so that each can be checked against a high-precision reference.  y, g*, res*, dz, dy*: NHWC
 * bf16 [rows][c]; c = 8, 16, 32, ..., 2048 (c / 8 must divide 256), rows > 0.  A CTA walks rows with lanes = 256 / (c/8)
 * row lanes per channel group; the column reductions write ONE fp32 row per CTA, partial [nblocks][K][c], at most
 * 4 x SMs rows (nblocks returned through nblocks_host).  Masks: [rows][c/8] bytes, bit j of byte (r, g) = element
 * (r, 8g + j) was > 0 after the ReLU. */

/* Slot 0 = sum y, slot 1 = sum y^2 (K = 2); dirb200_bn_finalize_layout with layout {nblocks, 1, c, 1} consumes them. */
int dirb200_layer_bn_stats(const void* y, int64_t rows, int c, float* partial, int* nblocks_host, void* stream);
/* out = [relu](fma(y, scale, shift) [+ res] [+ fma(res_y, res_scale, res_shift)]) in fp32, rounded once to bf16; at most
 * one of res / res_y.  mask_out (NULL: none; relu only) = the bits of the stored out. */
int dirb200_layer_bn_apply(const void* y, const float* scale, const float* shift, const void* res, const void* res_y,
                           const float* res_scale, const float* res_shift, int relu, int64_t rows, int c, void* out,
                           uint8_t* mask_out, void* stream);
/* BN backward moments.  dz = m * (g1 [+ g2] [+ g3]) summed in fp32 in that order; m = [fma(y, scale, shift) > 0] when
 * mask is NULL and scale / shift are given, the stored bit when mask is given, 1 when all three are NULL.  g2 / y2 /
 * dz_out / g3 need the mask; g3 needs g2 and dz_out; g2_h, g2_w > 0 (even, g2_h * g2_w dividing rows): g2 is the compact
 * [rows / (g2_h g2_w)][g2_h / 2][g2_w / 2][c] gradient added at even (y, x) of the g2_h x g2_w maps, not with y2.
 * dz_out (not with y2): dz rounded to bf16 and stored, the sums then taken over the stored values.  Slots: 0 = sum dz,
 * 1 = sum dz*y, 2 = sum dz*y2 (K = 3 with y2, else 2). */
int dirb200_layer_bn_bwd_reduce(const void* g1, const void* g2, const void* g3, const void* y, const void* y2,
                                const float* scale, const float* shift, const uint8_t* mask, int64_t rows, int c,
                                int g2_h, int g2_w, void* dz_out, float* partial, int* nblocks_host, void* stream);
/* From those rows (K = 2 or 3): dbeta = sum of slot 0, dgamma = invstd * (sum of slot gslot - mean * dbeta), both
 * ACCUMULATED into grad_gamma / grad_beta; coef_out [3][c] = A, B, C of dy = A*dz + B*y + C. */
int dirb200_layer_bn_bwd_coeffs(const float* partial, int nblocks, int k, int gslot, int64_t rows, int c,
                                const float* mean, const float* invstd, const float* gamma, float* grad_gamma,
                                float* grad_beta, float* coef_out, void* stream);
/* dy = bf16(fma(A, dz, fma(B, y, C))) with dz formed as in dirb200_layer_bn_bwd_reduce (no g3) and the coefficients
 * coef [3][c]; with y2, dy2 the same from (coef2, y2); dz_out (mask forms only, not with y2): dz stored.  g1 is dz
 * itself when mask, scale and shift are all NULL.  Compact g2 only together with dz_out. */
int dirb200_layer_bn_bwd_apply(const void* g1, const void* g2, const void* y, const float* coef, const void* y2,
                               const float* coef2, const float* scale, const float* shift, const uint8_t* mask,
                               int64_t rows, int c, int g2_h, int g2_w, void* dy, void* dy2, void* dz_out,
                               void* stream);
/* The stem's fused relu(bn(y)) + 3x3 / stride 2 / pad 1 max pool (c a multiple of 8): out = the pool of
 * bf16(relu(fma(y, scale, shift))), argmax = r*3+s of the first maximum in the window. */
int dirb200_layer_bn_relu_maxpool_fwd(const void* y, const float* scale, const float* shift, int n, int h, int w, int c,
                                      void* out, uint8_t* argmax, void* stream);
/* dirb200_maxpool3x3s2_bwd with a second gradient g2 of the pool output (NULL: none) added in fp32 to g1. */
int dirb200_layer_maxpool_bwd(const void* g1, const void* g2, const uint8_t* argmax, int n, int h, int w, int c,
                              void* dx, void* stream);

/* ------------------------------------------------ Test aids: the runner's batched kernels ---- */
/* The ResNet runner re-lays every conv weight, reduces every conv's split-K weight-gradient partials and forms every
 * eval-mode BatchNorm's coefficients with ONE launch over a descriptor table each.  These entry points run that launch
 * once over caller-given jobs, built with the runner's own descriptor construction, so that it can be checked against a
 * high-precision reference.  jobs_host is a HOST array of 1 .. 65535 jobs; the call copies it to a device table in
 * stream order (allocated, copied, launched and freed on `stream`).  Every argument is checked on the host before any
 * CUDA call: null pointers, non-positive sizes, negative offsets, a stem that is not 3x7x7 and a filter of 2^31 or more
 * weights (the index arithmetic divides 32-bit indices by multiply-high reciprocals) are refused. */

/* One conv: fp32 [cout][cin][kh][kw] at params + w_off -> w_fprop bf16 [cout][kh][kw][cin] and, when w_dgrad is not
 * NULL, w_dgrad bf16 [cin][kh][kw][cout] (round to nearest even).  stem (cin = 3, 7x7): w_fprop bf16 [cout][256] as
 * dirb200_conv_prep_weights(stem = 1) forms it; w_dgrad must be NULL. */
typedef struct dirb200_prep_job {
  int64_t w_off;
  int cout, cin, kh, kw, stem;
  void* w_fprop;
  void* w_dgrad;
} dirb200_prep_job;
int dirb200_prep_weights_all(const float* params, const dirb200_prep_job* jobs_host, int njobs, void* stream);

/* One conv: grads[w_off ..] fp32 [cout][cin][kh][kw] += sum over `splits` of the partials [splits][cout][kh*kw*cin]
 * (k = (r*kw + s)*cin + c, as the wgrad GEMM writes them); stem (cin = 3, 7x7): partials [splits][cout][256] over the
 * space-to-depth taps, the padding channel and the taps outside the 7x7 filter dropped. */
typedef struct dirb200_wgrad_reduce_job {
  const float* partial;
  int64_t w_off;
  int splits, cout, cin, kh, kw, stem;
} dirb200_wgrad_reduce_job;
int dirb200_wgrad_reduce_all(const dirb200_wgrad_reduce_job* jobs_host, int njobs, float* grads, void* stream);

/* One BatchNorm of c channels: scale = gamma * rsqrt(running_var + eps), shift = beta - running_mean * scale (fp32 [c]),
 * gamma / beta at params + gamma_off / beta_off, running_mean / running_var at running + rm_off / rv_off. */
typedef struct dirb200_bn_eval_job {
  int c;
  int64_t gamma_off, beta_off, rm_off, rv_off;
  float* scale;
  float* shift;
} dirb200_bn_eval_job;
int dirb200_bn_eval_coeffs_all(const dirb200_bn_eval_job* jobs_host, int njobs, const float* params,
                               const float* running, float eps, void* stream);

/* ------------------------------------------------ ResNet backbone runner ---- */
/* Opaque native runner of the bottleneck ResNet of agedb-dir/resnet.py:41-70,
 * 73-138 (conv1/bn1/relu/maxpool, layer1-4, avgpool, view) for one fixed
 * input shape.  It owns every activation / gradient / operand buffer (NHWC
 * bf16); parameters, their gradients and the BN running statistics stay in
 * caller-owned flat fp32 buffers laid out in the reference's
 * named_parameters() order: conv1.weight, bn1.weight, bn1.bias, then per
 * block conv1.weight, bn1.{weight,bias}, conv2.weight, bn2.*, conv3.weight,
 * bn3.*, [downsample.0.weight, downsample.1.{weight,bias}]; running stats per
 * BN in the same order as (running_mean, running_var). */
typedef struct dirb200_net dirb200_net;

/* H and W: multiples of 4 (the input space-to-depth needs even H, W; the max-pool backward an even stem output), at
 * most 1024 (the convolutions pack a stem-output row / column in 9 bits); N at most 8192 (13 bits of image index),
 * and N * H/2 * W/2 < 2^31. */
int dirb200_resnet_create(int n, int h, int w, const int* blocks_per_stage, int num_stages, dirb200_net** out);
void dirb200_resnet_destroy(dirb200_net* net);
int64_t dirb200_resnet_param_count(const dirb200_net* net);   /* floats in the flat parameter buffer */
int64_t dirb200_resnet_running_count(const dirb200_net* net); /* floats in the flat BN running buffer */
int64_t dirb200_resnet_feature_dim(const dirb200_net* net);   /* 2048 for ResNet-50 */
int64_t dirb200_resnet_device_bytes(const dirb200_net* net);

/* ResNet.forward up to `encoding` (resnet.py:128-138): x fp32 NCHW -> enc fp32
 * [n, feature_dim].  training: batch statistics + running-stat update. */
int dirb200_resnet_forward(dirb200_net* net, const float* x_nchw, const float* params, float* bn_running,
                           int training, float* enc_out, void* stream);

/* Backward of the above: d_enc fp32 [n, feature_dim]; ACCUMULATES into grads. */
int dirb200_resnet_backward(dirb200_net* net, const float* d_enc, const float* params, float* grads, void* stream);

/* The same backward, one stage per call, so that the caller can overlap the gradient all-reduce of a finished stage
 * (agedb-dir/train.py:143 DataParallel's reduction; SURVEY.md section 8e(1)) with the stages still running:
 * stage = dirb200_resnet_num_stages() (avg-pool backward + last layer group; reads d_enc), then stage-1 ... 1, then 0
 * (max-pool, stem).  In exactly that order after a training-mode forward.  dirb200_resnet_stage_param_range: the
 * [lo, hi) float range of the flat parameter / gradient buffers that stage owns (0 = conv1 + bn1). */
int dirb200_resnet_num_stages(const dirb200_net* net);
int dirb200_resnet_backward_stage(dirb200_net* net, int stage, const float* d_enc, const float* params, float* grads,
                                  void* stream);
int dirb200_resnet_stage_param_range(const dirb200_net* net, int stage, int64_t* lo, int64_t* hi);

/* Multi-scale encoder forward (nyud2-dir/models/modules.py:33-58, E_resnet.forward): the forward above without the
 * average pool; block_out[s] receives the output of the last block of layer group s+1 as NHWC bf16 [n, h_s, w_s, C_s]
 * (256 / 512 / 1024 / 2048 channels for ResNet-50).  training == 0: running statistics (folded-BN forward).  Every layer
 * group must end in an identity block (true of ResNet-50 and deeper). */
int dirb200_resnet_forward_blocks(dirb200_net* net, const float* x_nchw, const float* params, float* bn_running,
                                  int training, void* const* block_out, void* stream);

/* Its backward (nyud2-dir/models/modules.py:33-58, E_resnet.forward), one stage per call in the order of
 * dirb200_resnet_backward_stage: stage num_stages, ..., 1, then 0 (stem), after a training-mode forward.  Stage s >= 1
 * reads d_block, the NHWC bf16 gradient of block_out[s-1], or nothing when it is NULL; stage 0 reads nothing.
 * ACCUMULATES into grads, with the same per-stage parameter ranges.  A stage that receives no gradient, neither its own
 * nor from a stage above, does nothing (its parameter gradients keep their values). */
int dirb200_resnet_backward_blocks_stage(dirb200_net* net, int stage, const void* d_block, const float* params,
                                         float* grads, void* stream);

/* Per-kernel-class device timing of forward/backward (CUDA events around every launch group).  Classes:
 * 0 prep (weight re-layout, s2d), 1 conv fprop, 2 conv dgrad, 3 conv wgrad GEMM, 4 wgrad split-K reduce,
 * 5 BN statistics, 6 BN apply, 7 BN backward reduce, 8 BN backward apply, 9 pooling.
 * read_profile synchronises, fills ms_by_kind[10] / groups_by_kind[10] and clears the log. */
int dirb200_resnet_set_profiling(dirb200_net* net, int enabled);
int dirb200_resnet_read_profile(dirb200_net* net, double* ms_by_kind, int64_t* groups_by_kind);

/* Test / debugging aid: device pointer + shape ([rows][channels] bf16, NHWC) of an internal activation.
 * block = -1: stem (0 = conv1 raw, 1 = relu(bn1), 6 = max-pool output, 7 = max-pool argmax: u8 [rows][64], r*3 + s of
 * the window's first maximum); block >= 0: 0/1 = conv1 raw / act, 2/3 = conv2 raw / act, 4 = conv3 raw,
 * 5 = downsample raw, 6 = block output, 7 = the block output's ReLU mask: [rows][channels] bytes with
 * channels = C / 8, bit j of byte g = (output channel 8g + j > 0); refused unless the last forward was a training one.
 * A selector outside 0 .. 7, or 2 .. 5 for the stem, is refused before net is read. */
int dirb200_resnet_peek(dirb200_net* net, int block, int which, void** ptr, int64_t* rows, int* channels);

/* Test / debugging aid: one conv layer's own buffers and descriptor entries.  block = -1: the stem (conv 0);
 * block >= 0: conv 0 / 1 / 2 / 3 = conv1 / conv2 / conv3 / downsample.  w_fprop / w_dgrad: its bf16 GEMM operands
 * (w_dgrad NULL for the stem); partial: its split-K weight-gradient partials [splits][cout][kh*kw*cin] (stem:
 * [splits][cout][256]); scale / shift: its BatchNorm's fp32 [cout] coefficients; w_off: its weight's offset in the flat
 * parameter buffer; cout .. pad: the conv's hyper-parameters (stem: 3 -> cout, 7x7, stride 2, pad 3); splits: the
 * factor its entry in the runner's split-K reduction table holds (read back from the device: synchronises). */
typedef struct dirb200_conv_peek {
  void* w_fprop;
  void* w_dgrad;
  float* partial;
  float* scale;
  float* shift;
  int64_t w_off;
  int cout, cin, kh, kw, stride, pad, stem, splits;
} dirb200_conv_peek;
int dirb200_resnet_peek_conv(dirb200_net* net, int block, int conv, dirb200_conv_peek* out);

/* Test / debugging aid: the same conv's BatchNorm batch statistics, fp32 [cout] mean and invstd, as the last
 * training-mode forward left them (its own entry point: dirb200_conv_peek keeps its layout, which callers allocate). */
int dirb200_resnet_peek_bn_stats(dirb200_net* net, int block, int conv, float** mean, float** invstd);

/* nn.Linear(feature_dim, 1) (resnet.py:88,148): pred[n] = x[n,d] . w[d] + bias */
int dirb200_linear1_fwd(const float* x, const float* w, const float* bias, int64_t n, int d, float* pred,
                        void* stream);
/* dx[n,d] (may be NULL), dw[d], dbias[1] (all overwritten) */
int dirb200_linear1_bwd(const float* grad_pred, const float* x, const float* w, int64_t n, int d, float* dx,
                        float* dw, float* dbias, void* stream);

/* Fused optimizer steps over flat fp32 buffers (torch.optim.Adam / SGD semantics,
 * agedb-dir/train.py:163-164,262); grads are multiplied by grad_scale first
 * (1/world_size after a sum all-reduce) and, when clip_coef != NULL, by the device scalar *clip_coef
 * (dirb200_grad_clip_coef below: gradient-norm clipping without a host round trip). */
int dirb200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                      float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                      const float* clip_coef, void* stream);
int dirb200_sgd_step(float* params, const float* grads, float* momentum_buf, int64_t n, float lr, float momentum,
                     float weight_decay, int first_step, float grad_scale, const float* clip_coef, void* stream);

/* One tensor of a multi-tensor Adam step: four fp32 device buffers of numel elements (any 4-byte alignment; 16-byte
 * aligned ones are read with 128-bit accesses) and the tensor's own bias corrections for its step count t, computed by
 * the caller in double precision as dirb200_adam_step does: bc1 = 1 - beta1^t, bc2_sqrt = sqrt(1 - beta2^t), each
 * rounded to float. */
typedef struct dirb200_adam_segment {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t numel;
  float bc1;
  float bc2_sqrt;
} dirb200_adam_segment;

/* torch.optim.Adam with coupled L2 weight decay (no amsgrad, no maximize) over a list of tensors, the replacement of
 * torch.optim.Adam(model.parameters(), lr, weight_decay=1e-4) at nyud2-dir/train.py:146.  segs_host is a HOST array of
 * nseg segments; it is passed by value in the kernel's parameters (one launch per 512 segments), so the call copies
 * nothing to the device and the step is graph-capturable.  Per element the arithmetic is dirb200_adam_step's with
 * grad_scale 1, the parameter update written as one fma: exp_avg and exp_avg_sq get the same bits as the flat step,
 * a parameter may differ from it by about one ulp (the flat kernel's compiler fuses that update for some elements and
 * not for others). */
int dirb200_adam_step_multi(const dirb200_adam_segment* segs_host, int nseg, float lr, float beta1, float beta2,
                            float eps, float weight_decay, void* stream);
/* The same step with gradient-norm clipping, the replacement of clip_grad_norm(model.parameters(), max_grad_norm)
 * followed by optimizer.step() at sts-b-dir/trainer.py:147-150 (Adam, weight decay 1e-5, trainer.py:21): every
 * gradient is multiplied by the device scalar *clip_coef (dirb200_grad_norm_multi's out[0]) as it is read, and the
 * gradients are not rewritten.  Same kernel and arithmetic as dirb200_adam_step_multi: a coefficient of exactly 1
 * gives the same bits. */
int dirb200_adam_step_multi_clipped(const dirb200_adam_segment* segs_host, int nseg, float lr, float beta1,
                                    float beta2, float eps, float weight_decay, const float* clip_coef, void* stream);

/* One gradient of dirb200_grad_norm_multi: a 4-byte aligned fp32 device buffer of numel >= 0 elements (NULL when
 * empty). */
typedef struct dirb200_grad_segment {
  const float* grad;
  int64_t numel;
} dirb200_grad_segment;

/* torch.nn.utils.clip_grad_norm_'s norm and coefficient over a list of gradients (sts-b-dir/trainer.py:147-149,
 * --max_grad_norm): out[0] = min(1, max_norm / (||g||_2 + 1e-6)) (a NaN norm gives a NaN coefficient, as torch's
 * clamp), out[1] = ||g||_2 over every element of every segment.  segs_host is a HOST array passed by value in the
 * kernel parameters, one launch per 512 non-empty segments; the launches add into the workspace's fp64 partials and
 * the last one finalises.  Squares are summed in fp32 over at most 16 elements per thread, then in fp64; no
 * floating-point atomics, so two identical calls give identical bits.  The workspace (>= 8 KiB + 16 B, 8-byte
 * aligned) must be zero-initialised once; the kernel leaves its ticket word reset. */
size_t dirb200_grad_norm_multi_workspace_bytes(void);
int dirb200_grad_norm_multi(const dirb200_grad_segment* segs_host, int nseg, float max_norm, void* workspace,
                            size_t workspace_bytes, float* out, void* stream);

/* torch.nn.utils.clip_grad_norm_ over one flat gradient buffer (sts-b-dir/trainer.py:147-149, --max_grad_norm):
 * out[0] = min(1, max_norm / (||grad_scale * grads||_2 + 1e-6)), out[1] = that norm.  The gradients themselves are
 * not rewritten -- the optimizer step applies out[0] while it reads them.  workspace: >= 8 KiB + 16 B, fp64 partials. */
size_t dirb200_grad_clip_workspace_bytes(void);
int dirb200_grad_clip_coef(const float* grads, int64_t n, float grad_scale, float max_norm, void* workspace,
                           size_t workspace_bytes, float* out, void* stream);

/* ------------------------------------------- STS-B-DIR sentence-pair encoder ---- */
/* The 2-layer bidirectional LSTM of sts-b-dir/models.py:40-43 (nn.LSTM(d_word, d_hid, n_layers_enc,
 * bidirectional=True) run packed by the masked seq2seq wrapper) and the masked max-pool + pair features of
 * models.py:155-166.  Layouts and the gate interleaving are described in csrc/lstm.cu; rows M = 2B (s1 then s2),
 * lengths int32 in [1, T] (the caller checks), Hp / Dp the hidden / input sizes padded to multiples of 64.
 * T <= 4096, M <= 65535, Hp <= 4096. */
/* One layer's fp32 weights, both directions (torch layout, gate order i, f, g, o), -> bf16 GEMM operands:
 * w_ih [2*4Hp][Dp] (conv_fprop operand), w_ih_t [Dp][2*4Hp] (conv_dgrad operand), w_hh [2][4Hp][Hp],
 * w_hh_t [2][Hp][4Hp], bias fp32 [2][4Hp] = b_ih + b_hh.  The input has in_blocks blocks of din / in_blocks real
 * columns, each padded to Dp / in_blocks (layer 0: 1 block of d_word; later layers: the 2 directions' outputs).
 * Padding is zero. */
int dirb200_lstm_prep_weights(const float* w_ih_f, const float* w_hh_f, const float* b_ih_f, const float* b_hh_f,
                              const float* w_ih_r, const float* w_hh_r, const float* b_ih_r, const float* b_hh_r,
                              int H, int din, int in_blocks, int Hp, int Dp, void* w_ih, void* w_ih_t, void* w_hh,
                              void* w_hh_t, float* bias, void* stream);
/* Inverse of the re-layout for fp32 gradients: dw_ih [2*4Hp][Dp], dw_hh [2][4Hp][Hp], db [2][4Hp] -> the eight
 * torch-layout gradients (overwritten; db goes to both bias_ih and bias_hh). */
int dirb200_lstm_scatter_grads(const float* dw_ih, const float* dw_hh, const float* db, int H, int din, int in_blocks,
                               int Hp, int Dp, float* gw_ih_f, float* gw_hh_f, float* gb_ih_f, float* gb_hh_f,
                               float* gw_ih_r, float* gw_hh_r, float* gb_ih_r, float* gb_hh_r, void* stream);
/* Recurrent forward step s of both directions (one launch): gates = h_s . W_hh^T + xproj + bias, the cell update,
 * h_{s+1}, c_{s+1} and the output y at the step's time.  save != 0: h / c have T + 1 slots and the activated gates
 * (fp32) are kept for the backward; save == 0: 2 slots, gates unused.  dirb200_lstm_layer_fwd zeroes slot 0 and runs
 * every step, one launch each. */
int dirb200_lstm_fwd_step(const void* xproj, const void* w_hh, const float* bias, const int* lens, int T, int M,
                          int Hp, int save, int s, void* h, float* c, float* gates, void* y, void* stream);
int dirb200_lstm_layer_fwd(const void* xproj, const void* w_hh, const float* bias, const int* lens, int T, int M,
                           int Hp, int save, void* h, float* c, float* gates, void* y, void* stream);
/* Recurrent backward step s (one launch): dh = dgates_{s+1} . W_hh + dy at the step's time, the cell backward, the
 * pre-activation gradients dgates_s (bf16, step order dg [2][T][M][4Hp] and time order dg_time [T][M][2][4Hp]) and
 * the carried dc (fp32, dc [2][2][M][Hp]).  dirb200_lstm_layer_bwd runs s = T-1 .. 0. */
int dirb200_lstm_bwd_step(const void* w_hh_t, const void* dy, const float* gates, const float* c, const int* lens,
                          int T, int M, int Hp, int s, float* dc, void* dg, void* dg_time, void* stream);
int dirb200_lstm_layer_bwd(const void* w_hh_t, const void* dy, const float* gates, const float* c, const int* lens,
                           int T, int M, int Hp, float* dc, void* dg, void* dg_time, void* stream);
/* out[col] = sum over rows of bf16 x[rows][cols], fp32, in a fixed order (the LSTM bias gradient). */
int dirb200_col_sum_bf16(const void* x, int64_t rows, int cols, float* out, void* stream);
/* Embedding lookup (models.py:138, 141-142): x bf16 [T][M][Dp] = emb[ids[m][t]] * dmul[m][t] for t < lens[m], zero
 * elsewhere; ids int64 [M][T]; dmul fp32 [M][T][D] dropout multipliers or NULL. */
int dirb200_embed_gather(const int64_t* ids, const int* lens, const float* emb, const float* dmul, int64_t V, int M,
                         int T, int D, int Dp, void* x, void* stream);
/* Its gradient dw fp32 [V][D] (overwritten), deterministic: each row summed in position order m T + t.  Row
 * padding_index (-1: none) gets no gradient, as F.embedding's padding_idx; positions with an id outside [0, V)
 * contribute nothing. */
int dirb200_embed_grad(const int64_t* ids, const int* lens, const void* dx, const float* dmul, int64_t V, int M, int T,
                       int D, int Dp, int64_t padding_index, float* dw, void* stream);
/* Masked max over time and pair features (models.py:155-166): y bf16 [T][2B][2Hp] (layer output), dmul fp32
 * [2B][T][2H] or NULL -> feat fp32 [B][8H] = [u, v, |u - v|, u * v], arg int32 [2B][2H] the argmax time (first
 * maximal t on ties). */
int dirb200_pair_maxpool_fwd(const void* y, const int* lens, const float* dmul, int B, int T, int H, int Hp,
                             float* feat, int* arg, void* stream);
/* Its backward: dy bf16 [T][2B][2Hp] (zeroed here) gets the gradient at each argmax. */
int dirb200_pair_maxpool_bwd(const float* gfeat, const float* feat, const int* arg, const float* dmul, int B, int T,
                             int H, int Hp, void* dy, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIRB200_H */
