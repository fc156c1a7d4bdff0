/*
 * libstreamyolo_sm100.so -- C ABI of the H100-native StreamYOLO hot path.
 *
 * This is the drop-in boundary of SURVEY.md section 8(b): plain `extern "C"` entry
 * points, raw device pointers + sizes + a cudaStream_t, no torch types.  The host
 * side (streamyolo_b200/model/*.py, a mirror of the reference's exps/model API)
 * binds them with ctypes; INTEGRATION.md shows the stub a reference maintainer adds.
 *
 * Conventions
 *   - every function is asynchronous on `stream`, re-entrant, allocates nothing,
 *     never synchronises the device and never throws; it returns 0 or an SY_E*
 *     status and `sy_last_error_string()` describes the last failure of the
 *     calling thread.  The caller owns every buffer (PyTorch caching allocator).
 *   - activations are NHWC 16-bit "views" (SyTensor), bf16 unless an entry point says otherwise (SyConvDesc.storage,
 *     SyHeadPredDesc.storage, the *_f16 entry points): pixel (n,y,x) channel c lives
 *     at ptr + (((n*h + y)*w + x)*pitch + c) elements; pitch >= c lets a view be
 *     a channel slice of a wider concat buffer (pitch, slice offsets and c are
 *     multiples of 8 so that every pixel row is 16-byte aligned).
 *   - conv weights are bf16, packed [Cout][kh*kw][Cin] (K-major GEMM B operand).
 *   - the library requires an sm_90a device; there is no other code path.
 *
 * Each entry point cites the reference interface it replaces (paths relative to
 * /root/reference; "[yolox]" = the un-vendored yolox==0.3.0 dependency).
 */
#ifndef STREAMYOLO_SM100_H_
#define STREAMYOLO_SM100_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* sy_stream_t; /* == cudaStream_t */

enum {
  SY_OK = 0,
  SY_EINVAL = 1,   /* bad shape / alignment / null pointer */
  SY_EARCH = 2,    /* device is not sm_90 */
  SY_ELAUNCH = 3,  /* CUDA launch or driver error (see sy_last_error_string) */
  SY_EWORKSPACE = 4
};

/* 16-bit activation storage of a launch (SyConvDesc.storage, SyHeadPredDesc.storage) */
enum { SY_STORAGE_BF16 = 0, SY_STORAGE_F16 = 1 };

/* Activation after BatchNorm ([yolox] get_activation: "silu" / "relu" / "lrelu"), the `act` argument of sy_conv2d_tc,
 * sy_conv2d_simt, sy_dwconv2d (FUSED mode), sy_bn_act_apply and sy_bn_act_backward; any other value: SY_EINVAL.
 *   SY_ACT_NONE   identity
 *   SY_ACT_SILU   v * sigmoid(v)                    (nn.SiLU)
 *   SY_ACT_RELU   v > 0 ? v : 0                     (nn.ReLU;  derivative z > 0 ? 1 : 0)
 *   SY_ACT_LRELU  v > 0 ? v : 0.1f * v              (nn.LeakyReLU(0.1);  derivative z > 0 ? 1 : 0.1f)
 * The derivatives at z = 0 (0 for ReLU, 0.1 for LeakyReLU) are autograd's for the in-place modules yolox builds. */
enum { SY_ACT_NONE = 0, SY_ACT_SILU = 1, SY_ACT_RELU = 2, SY_ACT_LRELU = 3 };

typedef struct {
  void* ptr;      /* bf16 (fp16 where the entry point stores fp16) */
  int32_t n, h, w, c;
  int64_t pitch;  /* elements between consecutive pixels */
} SyTensor;

/* -------- runtime ---------------------------------------------------------- */
const char* sy_last_error_string(void);
int sy_version(void);
/* 0 when the current device is sm_90 and the driver exposes cuTensorMapEncodeTiled. */
int sy_check_device(void);

/* -------- convolution (replaces [yolox] BaseConv.conv / nn.Conv2d, e.g.
 * exps/model/darknet.py:115-165, exps/model/dfp_pafpn.py:33-105,
 * exps/model/tal_head.py:55-104) ------------------------------------------------- */
enum { SY_CONV_RAW = 0, SY_CONV_FUSED = 1 };

/* One BatchNorm parameter set covering output channels [c_begin, next segment's c_begin or Cout):
 * lets ONE conv launch serve two BaseConv modules that read the same input (CSPLayer conv1 | conv2). */
typedef struct {
  const float* gamma; const float* beta;          /* [c] */
  float* running_mean; float* running_var;        /* [c], updated in place (may be NULL) */
  int64_t* num_batches_tracked;                   /* += number of running-statistics updates (may be NULL) */
  int32_t c_begin;
} SyBnSegment;

typedef struct {
  SyTensor x;            /* input  */
  SyTensor y;            /* output: RAW -> conv result; FUSED -> act(acc*scale+shift)(+res) */
  const void* w;         /* bf16 [Cout][kh*kw][Cin] */
  int32_t kh, kw;        /* 1 or 3 each, padding (k-1)/2 */
  int32_t stride;        /* 1 or 2 */
  int32_t mode;          /* SY_CONV_RAW / SY_CONV_FUSED */
  int32_t act;           /* FUSED: SY_ACT_* (checked in every mode) */
  const float* scale;    /* FUSED: [Cout] (folded BatchNorm), may be NULL = 1 */
  const float* shift;    /* FUSED: [Cout], may be NULL = 0 */
  SyTensor res;          /* FUSED: optional residual added after the activation (ptr NULL = none) */
  /* ---- RAW mode: per-channel batch statistics of the stored output (sy_conv2d_tc only) ---- */
  int32_t split_n;       /* images >= split_n form statistics group 1 (0 or >= n: one group) */
  float* stat_partials;  /* [n_partials][Cout][2 groups][2 (sum, sumsq)] floats, one row per CTA (16B aligned), or NULL */
  int32_t n_partials;    /* >= sy_conv_stat_rows(); rows of CTAs that did not run are NOT written */
  int32_t* rows_written; /* out (host int, may be NULL): number of partial rows this launch writes */
  SyBnSegment bn[2];     /* bn[0].gamma != NULL: finalize BatchNorm in the kernel tail (1-2 parameter segments) */
  float momentum, eps;
  float* scale_shift;    /* [2 (scale|shift)][2 groups][Cout]: y = x*scale + shift, ready when the kernel ends */
  float* mean_invstd;    /* optional [2 (mean|invstd)][2 groups][Cout]: the batch statistics themselves, saved for
                          * sy_bn_act_backward (NULL: not written) */
  uint32_t* sync;        /* two zero-initialised counters (grid barrier + exit ticket); the kernel leaves them at zero.
                          * The normalise + act pass is sy_bn_act_apply, launched after the conv. */
  /* ---- debugging only: CTA 0 records (event, clock64) int64 pairs of its three pipeline roles ---- */
  void* debug_timeline;  /* device buffer of 2*debug_timeline_events int64, or NULL */
  int32_t debug_timeline_events;
  int32_t debug_flags;   /* 0 in production; 2 = skip TMA loads (pipeline dissection, results invalid); other values: SY_EINVAL */
  /* ---- validation only: the fp32 accumulators themselves, before the bf16 rounding of the stored result:
   * debug_f32[pixel][Cout] (pixel = flattened (n, oh, ow)), written next to the normal output.  This is where
   * north_star's "within 1e-3 of the reference" is literal (tests/test_gpu_ops.py::test_conv_fp32_accumulators). ---- */
  float* debug_f32;
  /* ---- tiling override (sy_conv2d_tc only; 0 = the planner's choice) ---- */
  int32_t tile_mode;     /* 1 = linear tiles, 2 = halo where the conv is 3x3 stride 1 (linear elsewhere); as SyConvPlan.mode */
  int32_t tile_bn;       /* tile width 64 or 128 */
  /* ---- running-statistics updates per statistics group (sy_conv2d_tc only) ---- */
  int32_t stat_updates;  /* 0 or 1: one update per group.  2: the launch's single group is folded into the running
                          * statistics twice, in the order and roundings of a two-group launch whose groups have equal
                          * statistics, and num_batches_tracked += 2 -- one pass over a batch that stands for two identical
                          * passes (a still frame duplicated into a pair).  Needs bn[] and one group; other values: SY_EINVAL */
  /* ---- activation storage (sy_conv2d_tc, sy_dwconv2d; sy_conv2d_simt takes bf16 only) ---- */
  int32_t storage;       /* SY_STORAGE_BF16 (0): x, y, res and w are bf16.  SY_STORAGE_F16 (1): all four are IEEE fp16
                          * (fp32 accumulation, one fp16 rounding of the stored result); FUSED mode only, without statistics,
                          * bn[] or the debug timeline (SY_EINVAL otherwise); debug_f32 works as with bf16 */
} SyConvDesc;

/* Rows of the statistics workspace (= SM count: one row per persistent CTA). */
int sy_conv_stat_rows(void);
/* wgmma implicit-GEMM kernel (TMA -> smem -> wgmma -> register accumulators -> epilogue).  In RAW mode with
 * stat_partials it also accumulates per-channel (sum, sum of squares) of the stored values per
 * statistics group, one partial row per CTA; with bn[] the persistent grid (all CTAs co-resident)
 * ends with a grid barrier and finalizes BatchNorm in parallel: batch statistics -> scale/shift,
 * running statistics (group 0 then group 1, unbiased variance, momentum).  Deterministic.  Do not
 * run two such launches concurrently on one GPU (the barrier needs every SM). */
int sy_conv2d_tc(const SyConvDesc* d, sy_stream_t stream);
/* Host-only query (no launch, no GPU needed): the tiling sy_conv2d_tc chooses for a layer shape and the descriptor's
 * tile_mode / tile_bn -- A-operand mode (1 linear tiles / im2col-mode TMA, 2 halo: 16 x 8 patches, the only mode with
 * patch_h x patch_w, else 0 x 0), tile width BN, tiles and rounds of the persistent grid, tile walk (0 N-major, 1 M-band:
 * each CTA keeps one N tile) and grid size. */
typedef struct SyConvPlan {
  int32_t mode, bn, m_tiles, n_tiles, rounds, kblocks, patch_h, patch_w, walk, grid;
} SyConvPlan;
int sy_conv2d_plan(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t kh, int32_t kw, int32_t stride,
                   int32_t tile_mode, int32_t tile_bn, SyConvPlan* out);
/* plain CUDA-core direct convolution with the same x/y/w/FUSED contract (no statistics):
 * device-side cross-check of the tensor-core kernel.  bf16 storage only (storage != 0: SY_EINVAL). */
int sy_conv2d_simt(const SyConvDesc* d, sy_stream_t stream);

/* Depthwise k x k convolution (groups = channels, k in {1, 3, 5}, stride 1 / 2): the first half of [yolox] DWConv, selected
 * by depthwise=True at exps/model/darknet.py:109, dfp_pafpn.py:31, tal_head.py:53.  Same descriptor and RAW / FUSED contract
 * as sy_conv2d_tc with x.c == y.c and w = bf16 [kh*kw][C]; the statistics fields are ignored (train-mode BatchNorm runs
 * through sy_channel_stats / sy_bn_finalize / sy_bn_act_apply).  Coalesced, vectorised CUDA-core kernel (HBM-bound).
 * storage = SY_STORAGE_F16: x, y, res and w fp16, FUSED mode only. */
int sy_dwconv2d(const SyConvDesc* d, sy_stream_t stream);

/* Focus stem, part 1: [yolox] Focus space-to-depth (TL/BL/TR/BR channel order), used at
 * exps/model/darknet.py:115.  x is the NCHW float32 frame-pair batch [b, in_ch, h, w]
 * (exps/model/dfp_pafpn.py:120,145 split it); image n of y takes frame n / b (0 = current,
 * 1 = support; channels 3*frame .. 3*frame+2) of batch element n % b.  y = [frames*b, h/2, w/2, 64]
 * bf16: for each focus pixel its three horizontal taps (x-1, x, x+1; zero outside the image), each
 * 12 focus channels + 4 zero channels, then 16 zero channels (one aligned 128-byte row per pixel).
 * The stem's 3x3 conv then runs on sy_conv2d_tc as a 3x1 conv over 64 channels with weights packed
 * [cout][3][64]. */
int sy_focus_pack(const float* x, int32_t b, int32_t in_ch, int32_t h, int32_t w_px, int32_t frames,
                  SyTensor y, sy_stream_t stream);
/* The same with y in fp16 (input pixels rounded to fp16), for the stem conv of an fp16-storage forward. */
int sy_focus_pack_f16(const float* x, int32_t b, int32_t in_ch, int32_t h, int32_t w_px, int32_t frames,
                      SyTensor y, sy_stream_t stream);

/* -------- BatchNorm (train mode) + activation (replaces nn.BatchNorm2d + nn.SiLU / ReLU / LeakyReLU inside
 * [yolox] BaseConv; eps/momentum from cfgs/s_s50_onex_dfp_tal_flip.py:40-44) ---------- */
/* Per-(row-chunk, channel) partial sums of a stored tensor: partials [P][2][c],
 * P = sy_stats_num_partials(n, h*w) image-major. */
int sy_stats_num_partials(int32_t n, int32_t hw);
int sy_channel_stats(SyTensor x, float* partials, int32_t n_partials, sy_stream_t stream);
/* Reduce partials per group (group 0 = partial rows [0,p_split), group 1 = the rest;
 * the two frames of a pair are normalised separately, exps/model/dfp_pafpn.py:120,145),
 * update running statistics sequentially group 0 then group 1 (unbiased variance,
 * momentum) and emit scale/shift [groups][c] with y = x*scale + shift. */
int sy_bn_finalize(const float* partials, int32_t n_partials, int32_t p_split, int32_t groups,
                   int64_t count_per_group, int32_t c,
                   const float* gamma, const float* beta, float* running_mean, float* running_var,
                   int64_t* num_batches_tracked, float momentum, float eps,
                   float* scale_out, float* shift_out, sy_stream_t stream);
/* y = act(x*scale[g]+shift[g]) (+ res), g = (image >= split_n), act = SY_ACT_*; single bf16 rounding.
 * y_group1_offset / res_group1_offset: element offsets added to the y / res addresses of the images of
 * statistics group 1 (0 = plain views).  The DFP fusion (exps/model/dfp_pafpn.py:168-170) uses them to
 * write jian(support frame n) into channels [c, 2c) of output image n - split_n, next to jian(current). */
int sy_bn_act_apply(SyTensor x, const float* scale, const float* shift, int32_t split_n, int32_t act,
                    SyTensor res, SyTensor y, int64_t y_group1_offset, int64_t res_group1_offset,
                    sy_stream_t stream);

/* -------- glue ------------------------------------------------------------- */
/* F.interpolate(mode="nearest", size=) of exps/model/dfp_pafpn.py:125,130 into a channel
 * slice; index rule src = min(floor(dst * (float)in/out), in-1) evaluated in float32. */
int sy_upsample_nearest(SyTensor x, SyTensor y, sy_stream_t stream);
/* [yolox] SPPBottleneck pooling (exps/model/darknet.py:156): y5,y9,y13 = stride-1
 * same-padded max pools (k = 5, 9, 13; -inf padding) of x. */
int sy_spp_maxpool(SyTensor x, SyTensor y5, SyTensor y9, SyTensor y13, sy_stream_t stream);
/* The same on fp16 views (the maximum of fp16 values: a different bit order from bf16). */
int sy_spp_maxpool_f16(SyTensor x, SyTensor y5, SyTensor y9, SyTensor y13, sy_stream_t stream);
/* strided copy of a view (used for 3-channel duplicates and buffers).  sy_upsample_nearest and sy_copy only move
 * 16-bit values, so they serve fp16 views unchanged. */
int sy_copy(SyTensor x, SyTensor y, sy_stream_t stream);
/* Per-stream first frame of a batched on_pipe tick: the star node of exps/model/dfp_pafpn.py:177-228 (no buffer: the
 * support features are the current ones, sup = cur) for the streams that start a sequence, the carried buffer for the
 * others.  For every image i with flags[i] != 0, image i of src[k] is copied into image i of dst[k], k < n_pairs (the
 * three FPN levels in ONE launch); images whose flag is clear are not touched.  The flags live in device memory, so a
 * CUDA graph that captured the launch follows what the host writes there before each replay.  Moves 16-bit values: bf16
 * and fp16 views alike. */
typedef struct {
  SyTensor src[3], dst[3];   /* pair k: [n][h][w][c] views of the same shape; pairs k >= n_pairs are ignored */
  int32_t n_pairs;           /* 1..3 */
  const int32_t* flags;      /* [n], device memory */
} SySelectImagesDesc;
int sy_select_images(const SySelectImagesDesc* d, sy_stream_t stream);

/* -------- head: prediction convs + decode (exps/model/tal_head.py:105-131,167-171,
 * 174,197-199,225-260) ------------------------------------------------------------ */
typedef struct {
  SyTensor cls_feat, reg_feat;   /* [b, h, w, c] */
  const float* w_reg; const float* b_reg;   /* [4][c], [4]  */
  const float* w_obj; const float* b_obj;   /* [1][c], [1]  */
  const float* w_cls; const float* b_cls;   /* [ncls][c], [ncls] */
  int32_t num_classes;
  int32_t stride;          /* 8 / 16 / 32 */
  int32_t anchor_offset;   /* first anchor row of this level in the [b, a_total, 5+ncls] output */
  int32_t a_total;
  int32_t sigmoid;         /* eval: sigmoid on obj / cls */
  int32_t decode;          /* xy = (xy + grid) * stride, wh = exp(wh) * stride */
  float* out;              /* [b, a_total, 5+ncls] float32 */
  float* origin;           /* [b, a_total, 4] raw reg (tal_head.py:185-194) or NULL */
  int32_t storage;         /* SY_STORAGE_BF16 (0): cls_feat / reg_feat are bf16; SY_STORAGE_F16 (1): fp16 */
} SyHeadPredDesc;
int sy_head_pred_decode(const SyHeadPredDesc* d, sy_stream_t stream);

/* -------- SimOTA + Trend-Aware loss (exps/model/tal_head.py:262-712) --------- */
typedef struct {
  int32_t b, a_total, max_labels, num_classes;
  int32_t n_levels;
  int32_t level_h[4], level_w[4], level_stride[4];
  const float* outputs;    /* [b, a_total, 5+ncls] decoded, logits for obj/cls */
  const float* origin;     /* [b, a_total, 4] raw reg */
  const float* labels_fut; /* [b, max_labels, 5] (cls, cx, cy, w, h) */
  const float* labels_cur; /* [b, max_labels, 5] */
  float gamma, ignore_thr, ignore_value;
  int32_t use_l1;
  void* workspace; size_t workspace_bytes;   /* >= sy_tal_loss_workspace_bytes() */
  float* loss_out;         /* [6]: total, 5*iou, obj(conf), cls, l1, num_fg / max(num_gt, 1) */
  /* optional dumps for tests / backward: */
  int32_t* fg_out;         /* [b, a_total] 0/1 or NULL */
  int32_t* matched_out;    /* [b, a_total] gt index or -1, or NULL */
  float* pred_iou_out;     /* [b, a_total] or NULL */
} SyTalLossDesc;
size_t sy_tal_loss_workspace_bytes(int32_t b, int32_t a_total, int32_t max_labels, int32_t num_classes);
int sy_tal_loss(const SyTalLossDesc* d, sy_stream_t stream);

/* Weight gradient of a convolution (the cuDNN backward-filter call behind loss.backward(),
 * exps/train_utils/double_trainer.py:114, for every [yolox] BaseConv: exps/model/darknet.py:115-165,
 * dfp_pafpn.py:33-105, tal_head.py:55-104):  dw[co][ci][r][s] (+)= sum_p dy[p][co] * x[p @ (r, s)][ci].
 * x = the layer's input [n, h, w, cin] bf16, dy = gradient w.r.t. the conv output [n, ho, wo, cout] bf16 (same kernel
 * size / stride / padding (k-1)/2 as the forward), dw = fp32 in PyTorch's OIHW parameter layout.  Split-K over the
 * pixels on the tensor cores, then a fixed-order reduction (deterministic).  The workspace holds the fp32 partials. */
typedef struct SyConvWgradDesc {
  SyTensor x;
  SyTensor dy;
  int32_t kh, kw, stride;
  float* dw;               /* [cout, cin, kh, kw] fp32 */
  int32_t accumulate;      /* 0: dw = result, 1: dw += result */
  void* workspace;         /* sy_conv2d_wgrad_workspace_bytes(desc) bytes, 16-byte aligned */
  size_t workspace_bytes;
} SyConvWgradDesc;
size_t sy_conv2d_wgrad_workspace_bytes(const SyConvWgradDesc* d);
int sy_conv2d_wgrad_tc(const SyConvWgradDesc* d, sy_stream_t stream);

/* Backward of BatchNorm(train) + activation behind a [yolox] BaseConv (autograd of nn.BatchNorm2d + the act module under
 * loss.backward(), exps/train_utils/double_trainer.py:114).  raw = the conv output the forward stored, dy = gradient w.r.t.
 * the BaseConv output; scale / shift / mean / invstd = [2 groups][c] as published by the forward (scale = gamma * invstd,
 * shift = beta - mean * scale; images >= split_n form statistics group 1).  Writes draw (bf16, gradient w.r.t. the conv
 * output, input of the conv data / weight gradient kernels), dgamma / dbeta (fp32, (+)=).  partials: sy_bn_act_bwd_rows(n,
 * h*w) rows of 2*c floats; coef: 8*c floats of scratch. */
typedef struct SyBnActBwdDesc {
  SyTensor raw, dy, draw;
  const float* scale; const float* shift; const float* mean; const float* invstd;
  int32_t split_n;
  int32_t act;             /* SY_ACT_* of the forward */
  float* dgamma; float* dbeta;
  int32_t accumulate;
  float* partials; int32_t n_partials;
  float* coef;
} SyBnActBwdDesc;
int sy_bn_act_bwd_rows(int32_t n, int32_t hw);
int sy_bn_act_backward(const SyBnActBwdDesc* d, sy_stream_t stream);

/* Zero-insertion D[n, 2i, 2j, :] = g[n, i, j, :] (D = [n, H, W, c], H in {2h-1, 2h}): the data gradient of a stride-2
 * 3x3 conv (the first convs of dark2..dark5, bu_conv1/2: exps/model/darknet.py:118-160, dfp_pafpn.py:57-69) is then
 * sy_conv2d_tc on D with the flipped, channel-transposed filter, stride 1. */
int sy_dilate2(SyTensor g, SyTensor D, sy_stream_t stream);

/* Backward of F.interpolate(mode="nearest") (exps/model/dfp_pafpn.py:126,131): dx[n, iy, ix] = sum of dy over the
 * destination pixels whose source index (the forward's fp32 expression) is (iy, ix). */
int sy_upsample_nearest_backward(SyTensor dy, SyTensor dx, sy_stream_t stream);

/* y += x (bf16): gradient accumulation where a tensor feeds several consumers (Bottleneck shortcuts,
 * exps/model/dfp_pafpn.py:168-170 "+ cur", FPN features read by two branches). */
int sy_add(SyTensor x, SyTensor y, sy_stream_t stream);

/* Backward of the three SPP max pools ([yolox] SPPBottleneck, exps/model/darknet.py:156): dx = gradient reaching x
 * through MaxPool2d(5), (9), (13) (stride 1, padding k/2), each window's gradient going to its first maximum in
 * row-major order like PyTorch.  The identity branch of the concat is not included.  Deterministic (gather). */
size_t sy_spp_maxpool_backward_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t c);
int sy_spp_maxpool_backward(SyTensor x, SyTensor d5, SyTensor d9, SyTensor d13, SyTensor dx, void* workspace,
                            size_t workspace_bytes, sy_stream_t stream);

/* Backward of the three 1x1 prediction convs of one head level (exps/model/tal_head.py:101-131, 163-171):
 * grad_raw [b, a_total, 5 + nc] (d loss / d raw head outputs, sy_tal_loss_backward) -> gradients w.r.t. the cls / reg
 * tower outputs (bf16 views), the conv weights ([4][c], [1][c], [nc][c]) and biases (fp32, (+)=).
 * partials: sy_head_pred_bwd_rows(b, h, w) rows of (5 + nc) * (c + 1) floats. */
typedef struct SyHeadPredBwdDesc {
  const float* grad_raw;
  SyTensor cls_feat, reg_feat;         /* the forward's inputs */
  SyTensor d_cls_feat, d_reg_feat;     /* outputs */
  const float* w_reg; const float* w_obj; const float* w_cls;
  int32_t num_classes, a_total, anchor_offset;
  float* dw_reg; float* dw_obj; float* dw_cls; float* db_reg; float* db_obj; float* db_cls;
  int32_t accumulate;
  float* partials; int32_t n_partials;
} SyHeadPredBwdDesc;
int sy_head_pred_bwd_rows(int32_t b, int32_t h, int32_t w);
int sy_head_pred_backward(const SyHeadPredBwdDesc* d, sy_stream_t stream);
/* The same backward for 1 <= num_classes <= 251 with (5 + num_classes) * c * 4 <= 200 KiB, the limits of
 * sy_head_pred_decode (what the reference's TALHead / PIPEHead take, exps/model/tal_head.py:27, 101-131, 163-171, under
 * loss.backward(), exps/train_utils/double_trainer.py:114).  Same descriptor, same partials (sy_head_pred_bwd_rows rows),
 * fixed-order reduction: deterministic.  sy_head_pred_backward keeps its 27-class limit; the trainer uses this entry
 * point above it. */
int sy_head_pred_backward_wide(const SyHeadPredBwdDesc* d, sy_stream_t stream);

/* Backward of the loss: what autograd computes for loss.backward() (exps/train_utils/double_trainer.py:114)
 * through TALHead.get_losses (exps/model/tal_head.py:426-461): the SimOTA assignment, the class targets and the
 * normalised TAL weights are constants (tal_head.py:479 @torch.no_grad, weights detached), so the gradient is
 * per anchor.  Must run after sy_tal_loss on the SAME workspace (assignment and loss sums are read from it).
 * grad_outputs: d/d outputs[b, a, :] (decoded boxes, obj / cls logits); grad_origin: d/d origin_preds;
 * grad_raw: d/d the raw head-conv outputs, i.e. the decode of tal_head.py:237-241 folded in and the L1 path added
 * (what the prediction convs' backward consumes).  Any of the three may be NULL. */
typedef struct SyTalLossBwdDesc {
  const float* outputs;    /* [b, a_total, 5 + num_classes] as given to sy_tal_loss */
  const float* origin;     /* [b, a_total, 4] or NULL when !use_l1 */
  const float* labels_fut; /* [b, max_labels, 5] */
  int32_t b, a_total, max_labels, num_classes, n_levels;
  int32_t level_h[4], level_w[4], level_stride[4];
  float gamma;
  int32_t use_l1;
  void* workspace;         /* the workspace sy_tal_loss ran on */
  size_t workspace_bytes;
  float grad_scale;        /* d objective / d total_loss (1, or the AMP loss scale) */
  float* grad_outputs;     /* [b, a_total, 5 + num_classes] or NULL */
  float* grad_origin;      /* [b, a_total, 4] or NULL */
  float* grad_raw;         /* [b, a_total, 5 + num_classes] or NULL */
} SyTalLossBwdDesc;
int sy_tal_loss_backward(const SyTalLossBwdDesc* d, sy_stream_t stream);

/* Detection post-processing = [yolox 0.3.0] yolox.utils.postprocess as called by the evaluators and the streaming
 * driver (exps/evaluators/onex_stream_evaluator.py:148, sAP/streamyolo/streamyolo_det.py:62-83): cxcywh -> xyxy,
 * class_conf / class_pred = max over the class scores, keep obj * class_conf >= conf_thre, class-aware greedy NMS
 * (torchvision.ops.batched_nms semantics), rows [x1, y1, x2, y2, obj, class_conf, class_pred] in decreasing score order.
 * pred = the eval-mode head output [b, a_total, 5 + num_classes] (decoded boxes, sigmoid scores).  One CTA per image;
 * a_total <= 16384.  det_out [b, max_det, 7] (rows past count_out[i] are not written), count_out [b]. */
typedef struct SyNmsDesc {
  const float* pred;
  int32_t b, a_total, num_classes, max_det;
  float conf_thre, nms_thre;
  int32_t class_agnostic;
  void* workspace;         /* sy_postprocess_nms_workspace_bytes(b, a_total) bytes, 16-byte aligned */
  size_t workspace_bytes;
  float* det_out;
  int32_t* count_out;
} SyNmsDesc;
size_t sy_postprocess_nms_workspace_bytes(int32_t b, int32_t a_total);
int sy_postprocess_nms(const SyNmsDesc* d, sy_stream_t stream);

/* Per-stream gating of a batched streaming tick whose frames were decoded on the device (sy_jpeg_decode_sized): the
 * driver's loop (sAP/streamyolo/streamyolo_det.py:150-195) only runs the model on a frame it has.  For every stream i,
 * start[i] = (status[i] == SY_JPEG_OK && flags[i] != 0) and keep[i] = (status[i] == SY_JPEG_OK); status NULL counts every
 * stream as decoded.  start feeds sy_select_images' first-frame choice and keep the buffer update, so a stream without a
 * decoded frame keeps its carried features.  All arrays [n] int32 in device memory; no host synchronisation. */
int sy_stream_gate(const int32_t* status, const int32_t* flags, int32_t n, int32_t* start, int32_t* keep, sy_stream_t stream);
/* Per-stream box rescale of sy_postprocess_nms' rows, replacing the host's `detections[:, :4] / in_scale` of the driver's
 * inference() (streamyolo_det.py:82) and the evaluators' `bboxes /= scale` (exps/evaluators/onex_stream_evaluator.py:182):
 * det [n][max_det][7], rows < count[i] of stream i get x1, y1, x2, y2 divided by ratio[i] (fp32, IEEE division), and
 * count[i] = 0 where status[i] != SY_JPEG_OK (status may be NULL). */
int sy_stream_rescale(float* det, int32_t n, int32_t max_det, int32_t* count, const int32_t* status, const float* ratio,
                      sy_stream_t stream);
/* Device half of the validation evaluators' convert_to_coco_format (exps/evaluators/onex_stream_evaluator.py:167-209,
 * twox_stream_evaluator.py:165-217, still_stream_evaluator.py:137-169) for a batch of b images: the first count[i] rows
 * of image i of sy_postprocess_nms' det [b][max_det][7] become COCO detection rows, compacted image-major in NMS order:
 * bbox_out [N][4] = x1 / r, y1 / r, x2 / r - x1 / r, y2 / r - y1 / r (`bboxes /= scale; xyxy2xywh(bboxes)`, fp32, one
 * rounding per operation, r = ratio[i]), score_out [N] = obj * class_conf (fp32), category_out [N] =
 * class_ids[(int)class_pred] (-1 for a class outside [0, num_classes)), image_id_out [N] = image_id[i], and
 * total_out [1] = N.  An image emits nothing when image_id[i] < 0 (the evaluator's frame-id rules drop it), or, with
 * status given, when any of its frames_per_image frames status[i * frames_per_image + f] is not SY_JPEG_OK.  The outputs
 * hold room for b * max_det rows; rows past N are not written.  All arrays in device memory; b <= 4096. */
typedef struct SyCocoRowsDesc {
  const float* det;
  int32_t b, max_det;
  const int32_t* count;        /* [b] */
  const float* ratio;          /* [b] */
  const int32_t* image_id;     /* [b], < 0: emit nothing */
  const int32_t* status;       /* [b * frames_per_image] SY_JPEG_*, or NULL */
  int32_t frames_per_image;
  int32_t num_classes;
  const int32_t* class_ids;    /* [num_classes] */
  float* bbox_out;
  float* score_out;
  int32_t* image_id_out;
  int32_t* category_out;
  int32_t* total_out;
} SyCocoRowsDesc;
int sy_coco_rows(const SyCocoRowsDesc* d, sy_stream_t stream);

/* -------- forecast (streamyolo_b200/csrc/forecast.cu) ----------------------------------------------------------------
 * The sAP toolkit's forecast of streaming detections to the query frame (sAP/forecast/pps_forecast_kf.py with
 * --forecast-before-assoc and --assoc iou): on every new detection a constant-velocity Kalman predict of the tracks
 * (F(dt), Q = dt^2 I, :175-184), greedy IoU association of the score-sorted detections with the tracks
 * (sAP/track/__init__.py:90-133, no_unmatched1, pycocotools' fp64 bbIou, ties to the later track) and a Kalman update of
 * the matched ones (R = 10 I, :81-97); at a query, the matched tracks extrapolated dt frames ahead and every track
 * cleaned up by extrap_clean_up(..., lt=True) (sAP/forecast/__init__.py:33-56, min_size 75).  One CTA per stream or
 * sequence; the state lives in caller-owned device buffers of S streams of at most T tracks.  Every entry point is
 * capturable: no allocation, no synchronisation. */
typedef struct SyForecastState {
  float* x;          /* [S][T][8] Kalman mean: l, t, w, h and their velocities */
  float* P;          /* [S][T][8][8] covariance */
  int32_t* label;    /* [S][T] */
  float* score;      /* [S][T] */
  int32_t* track;    /* [S][T] track id */
  int32_t* meta;     /* [S][4]: n_tracks, n_matched, next track id, overflow (set when a detection had more than T rows;
                        that stream's state is then left as it was) */
  int32_t S, T;      /* 1 <= S <= 65535, 1 <= T <= 2^20 */
} SyForecastState;
/* scratch bytes of sy_forecast_update / sy_forecast_sequences for S streams (sequences) of at most T tracks */
size_t sy_forecast_workspace_bytes(int32_t streams, int32_t max_tracks);
/* One new detection per stream (pps_forecast_kf.py:167-256): det [S][max_det][7] and count [S] as sy_postprocess_nms
 * and sy_stream_rescale leave them (score = obj * class_conf, label = (int)class_pred); dt [S] the frames between this
 * detection's input frame and the previous one's; start [S] (or NULL) != 0 clears the stream's tracks and restarts its
 * track ids at 0 first; keep [S] (or NULL) == 0 leaves the stream untouched.  A new detection with no rows keeps the
 * predicted tracks and n_matched (pps_forecast_kf.py), or, with clear_on_empty != 0, leaves the stream without tracks
 * (sAP/forecast/streamer.py:247-280); the track id counter continues either way. */
typedef struct SyForecastUpdateDesc {
  SyForecastState state;
  const float* det;
  int32_t max_det;
  const int32_t* count;
  const int32_t* dt;
  const int32_t* start;
  const int32_t* keep;
  double match_iou_th;     /* inclusive */
  void* workspace;
  size_t workspace_bytes;
  int32_t clear_on_empty;  /* 0: pps_forecast_kf.py's rule for an empty detection; else streamer.py's */
} SyForecastUpdateDesc;
int sy_forecast_update(const SyForecastUpdateDesc* d, sy_stream_t stream);
/* Each stream's tracks extrapolated dt[s] frames ahead (:258-273): the first n_matched as x[:4] + dt * x[4:], the others
 * as x[:4]; then extrap_clean_up with the stream's image size img_wh[s] = (W, H).  Rows compacted in track order at
 * [s][0..count_out[s]) of box_out [S][T][4] (l, t, w, h), score_out, label_out, track_out [S][T]. */
typedef struct SyForecastExtrapDesc {
  SyForecastState state;
  const int32_t* dt;       /* [S] */
  const int32_t* img_wh;   /* [S][2] */
  float* box_out;
  float* score_out;
  int32_t* label_out;
  int32_t* track_out;
  int32_t* count_out;      /* [S] */
} SyForecastExtrapDesc;
int sy_forecast_extrap(const SyForecastExtrapDesc* d, sy_stream_t stream);
/* Up to Q queries per stream in one launch: stream s's tracks extrapolated dt[s][k] frames ahead for k < n_query[s], each
 * as sy_forecast_extrap does with an fp32 dt (the streamer's fractional query, sAP/forecast/streamer.py:287-297: numpy's
 * fp32 x[:4] + dt * x[4:]); an integer dt gives sy_forecast_extrap's rows bit for bit.  Query (s, k) writes its rows at
 * [s][k][0..count_out[s][k]) of box_out [S][Q][T][4] (l, t, w, h), score_out, label_out, track_out [S][Q][T];
 * count_out [S][Q] is 0 for k >= n_query[s]. */
typedef struct SyForecastExtrapQueriesDesc {
  SyForecastState state;
  const float* dt;         /* [S][Q] */
  const int32_t* n_query;  /* [S] */
  int32_t Q;               /* 1 <= Q <= 65535 */
  const int32_t* img_wh;   /* [S][2] */
  float* box_out;
  float* score_out;
  int32_t* label_out;
  int32_t* track_out;
  int32_t* count_out;      /* [S][Q] */
} SyForecastExtrapQueriesDesc;
int sy_forecast_extrap_queries(const SyForecastExtrapQueriesDesc* d, sy_stream_t stream);
/* The offline pass (pps_forecast_kf.py:134-287) over S sequences, one CTA each, with the state of sy_forecast_update
 * (cleared at each sequence's start).  Detection k has det_n[k] rows at det + 7 * det_start[k] (rows as in
 * sy_forecast_update).  Sequence s owns the frames [seq_frames[s], seq_frames[s + 1]) of frames [F][6]: (index of the
 * latest detection or -1, dt of the update when that detection is new, dt of the query, first output row, W, H).  A
 * frame's rows go to its first output row on (room for its track count, which the host knows) and rows_out [F] counts
 * them; a frame without a detection, or whose sequence has no track yet, emits nothing. */
typedef struct SyForecastSequencesDesc {
  SyForecastState state;
  const float* det;
  const int32_t* det_start;
  const int32_t* det_n;
  const int32_t* frames;
  const int32_t* seq_frames;   /* [S + 1] */
  double match_iou_th;
  float* box_out;
  float* score_out;
  int32_t* label_out;
  int32_t* track_out;
  int32_t* rows_out;           /* [F] */
  void* workspace;
  size_t workspace_bytes;
} SyForecastSequencesDesc;
int sy_forecast_sequences(const SyForecastSequencesDesc* d, sy_stream_t stream);

/* -------- training step glue (streamyolo_b200/csrc/train_glue.cu) ---------------------------------------------- */
/* fp32 OIHW conv parameter -> bf16 GEMM operand, on the device (one launch per parameter per optimiser step):
 *   mode 0  out[o][r*kw+s][i] = w[o][i][r][s]                          forward B operand of sy_conv2d_tc
 *   mode 1  out[i][taps-1-(r*kw+s)][co_offset + o] = w[o][i][r][s]     data-gradient operand (flipped taps, transposed
 *           channels; rows of out_pitch elements so that the conv1 | conv2 pair of a CSPLayer packs into one operand)
 *   mode 2  out[o][r][s*16 + i] = w[o][i][r][s], 64 columns per (o, r) Focus stem (see sy_focus_pack)
 *   mode 0 | SY_PACK_F16, mode 2 | SY_PACK_F16: the same layouts in fp16 (operands of fp16-storage forwards)
 * Replaces the weight.to(bf16).permute chain a PyTorch host would run after every optimizer.step()
 * (exps/train_utils/double_trainer.py:119-121). */
enum { SY_PACK_F16 = 0x100 };
int sy_pack_conv_weight(const float* w, int32_t cout, int32_t cin, int32_t kh, int32_t kw, int32_t mode, void* out,
                        int64_t out_pitch, int32_t co_offset, sy_stream_t stream);

/* The same for MANY parameters in one launch: items (a DEVICE array) lists (parameter, layout) pairs with the arguments of
 * sy_pack_conv_weight.  The launch works in TILES (64 output x 32 input channels of one item; 64 output channels of a stem
 * item): `begin` = index of the item's first tile (prefix sum of sy_pack_item_tiles over the items), `total` = their sum.
 * The trainer re-packs every conv operand of the model (forward and data-gradient layouts) with it after each optimiser step. */
typedef struct SyPackItem {
  const float* w;
  void* out;
  int32_t cout, cin, kh, taps, mode, co_offset;
  int64_t out_pitch;
  int64_t begin;
} SyPackItem;
int64_t sy_pack_item_tiles(int32_t cout, int32_t cin, int32_t mode);
int sy_pack_conv_weights_batch(const SyPackItem* items_dev, int32_t n_items, int64_t total, sy_stream_t stream);

/* The optimiser step of the reference trainer as one launch over flat fp32 state (SURVEY section 8 f3):
 * GradScaler.unscale_ + [yolox] Exp.get_optimizer's SGD(momentum, nesterov) with weight decay on the conv / linear weights
 * only + [yolox] ModelEMA.update (exps/train_utils/double_trainer.py:113-123, 173-175).  Elements [0, n_param) are
 * parameters in the order (BatchNorm weights, biases | decayed weights from decay_begin); [n_param, n_total) are the
 * floating-point buffers (BatchNorm running statistics) that only the EMA follows.  Step-by-step the same roundings as
 * torch.optim.SGD / ModelEMA in fp32.  found_inf (device float, may be NULL): non-zero skips the whole update, or with
 * found_inf_ema non-zero only the parameter and momentum update: the EMA still runs ema = d * ema + (1 - d) * param, as
 * ModelEMA.update does after a step GradScaler skipped (double_trainer.py:115-119). */
typedef struct SySgdEmaDesc {
  float* param;              /* [n_total] model state (parameters then float buffers) */
  const float* grad;         /* [n_param] (the all-reduced flat gradient buffer) */
  float* momentum_buf;       /* [n_param] */
  float* ema;                /* [n_total] or NULL (no EMA) */
  int64_t n_param, n_total, decay_begin;
  float lr, momentum, weight_decay, inv_scale;
  int32_t nesterov;
  float ema_decay, ema_one_minus_decay;
  const float* found_inf;
  /* optional device array [lr, momentum, weight_decay, inv_scale, ema_decay, 1 - ema_decay]: when non-NULL it REPLACES the
   * six scalars above, so that a step captured in a CUDA graph follows the LR schedule / EMA ramp / loss scale of the
   * iteration it is replayed in (the host rewrites the 24 bytes before each replay). */
  const float* hyper;
  int32_t found_inf_ema;     /* 0: a non-zero *found_inf skips the EMA too; else the EMA still runs (see above) */
} SySgdEmaDesc;
int sy_sgd_nesterov_ema_step(const SySgdEmaDesc* d, sy_stream_t stream);

/* GradScaler's inf / NaN check of the gradients (torch._amp_foreach_non_finite_check_and_unscale_, behind
 * GradScaler.step at exps/train_utils/double_trainer.py:115), over one flat fp32 buffer x[0, n) (16-byte aligned):
 * *flag = 1.0 if any element is NaN or +-inf, else 0.0, and *count += 1 when it is 1.0 (a device counter of skipped
 * steps).  The flag is reset by this call (a memset, then one vectorised pass), so it can be captured in a CUDA graph and
 * replayed.  flag then goes to SySgdEmaDesc.found_inf. */
int sy_nonfinite_flag(const float* x, int64_t n, float* flag, int32_t* count, sy_stream_t stream);

/* Input pipeline on the device (SURVEY section 8 f4): Exp.preprocess (cfgs/s_s50_onex_dfp_tal_flip.py:160-171) =
 * F.interpolate(inputs, size=tsize, mode="bilinear", align_corners=False) on the NCHW fp32 frame-pair batch
 * (x: [nc = B*6][hi][wi] -> y: [nc][ho][wo]) and the label rescale targets[..., 1::2] *= sx, [..., 2::2] *= sy
 * (labels: rows x cols floats, column 0 = class, in place). */
int sy_resize_bilinear(const float* x, int32_t nc, int32_t hi, int32_t wi, float* y, int32_t ho, int32_t wo,
                       sy_stream_t stream);
int sy_scale_labels(float* labels, int64_t rows, int32_t cols, float sx, float sy, sy_stream_t stream);

/* -------- input transforms (streamyolo_b200/csrc/input.cu) ------------------------------------------------------ */
/* Label half of DoubleTrainTransform(max_labels, hsv=False, flip) (exps/data/data_augment_flip.py:141-148, 176-234) for
 * n_items frame pairs, one warp per frame, in fp64 with one final cast to fp32: mirror the boxes (x1' = width - x2,
 * x2' = width - x1) when flip && mirror[item] && the frame has rows, xyxy -> cxcywh, * r, keep rows with min(w, h) > 1;
 * if none survive, the unmirrored, unfiltered rows instead.  Rows past max_labels are dropped, the rest is zero.
 * flags_out receives each frame's effective mirror bit, which sy_letterbox reads: launch this first on the same stream. */
typedef struct SyPairLabelsDesc {
  const double* ann;       /* [n_items][2][max_rows][5] x1, y1, x2, y2, cls (frame 0 = current image, future boxes) */
  const int32_t* counts;   /* [n_items][2] valid rows of each frame (clamped to [0, max_rows]) */
  const int32_t* mirror;   /* [n_items] the pair's mirror bit (may be NULL when flip == 0) */
  int32_t n_items, max_rows, max_labels, flip;
  int32_t width;           /* width of the frame entering the transform: the mirror axis */
  double r;                /* letterbox scale min(H / h, W / w) */
  float* labels_fut;       /* [n_items][max_labels][5] cls, cx, cy, w, h of frame 0 */
  float* labels_cur;       /* [n_items][max_labels][5] of frame 1 */
  int32_t* flags_out;      /* [n_items][2] */
} SyPairLabelsDesc;
int sy_pair_labels(const SyPairLabelsDesc* d, sy_stream_t stream);

/* The same for n independent frames: the label half of TrainTransform(max_labels, hsv=False, flip)
 * (exps/data/data_augment_flip.py:170-234), the dataset transform of the still-image baseline.  Per frame the rules of
 * sy_pair_labels; flags_out[i] is frame i's effective mirror bit for sy_letterbox over the same n frames. */
typedef struct SyFrameLabelsDesc {
  const double* ann;       /* [n][max_rows][5] x1, y1, x2, y2, cls */
  const int32_t* counts;   /* [n] valid rows (clamped to [0, max_rows]) */
  const int32_t* mirror;   /* [n] mirror bits (may be NULL when flip == 0) */
  int32_t n, max_rows, max_labels, flip;
  int32_t width;           /* width of the frame entering the transform: the mirror axis */
  double r;                /* letterbox scale min(H / h, W / w) */
  float* labels;           /* [n][max_labels][5] cls, cx, cy, w, h */
  int32_t* flags_out;      /* [n] */
} SyFrameLabelsDesc;
int sy_frame_labels(const SyFrameLabelsDesc* d, sy_stream_t stream);

/* Image half: uint8 HWC BGR frames [n][h][w][3] -> fp32 planar [n][3][out_h][out_w] (a [B][6][H][W] pair batch when
 * n = 2B).  Each frame goes through cv2.resize(INTER_LINEAR) h x w -> mid_h x mid_w (load_resized_img,
 * exps/dataset/tal_flip_one_future_argoversedataset.py:179-187; none when mid == h x w), the mirror when flags[i] is
 * set, cv2.resize mid -> dst_h x dst_w (preproc, data_augment_flip.py:151-167; none when dst == mid), top-left on a canvas
 * of 114, bit-identical to OpenCV's 8-bit fixed-point bilinear resize.  With dst == out and no flags it is the streaming
 * driver's preproc (sAP/streamyolo/streamyolo_det.py:57-60, 176-181). */
typedef struct SyLetterboxDesc {
  const uint8_t* src;      /* [n][h][w][3] */
  int32_t n, h, w;
  int32_t mid_h, mid_w;
  int32_t dst_h, dst_w;
  int32_t out_h, out_w;
  const int32_t* flags;    /* [n] mirror bits, or NULL */
  float* out;              /* [n][3][out_h][out_w] */
} SyLetterboxDesc;
int sy_letterbox(const SyLetterboxDesc* d, sy_stream_t stream);
/* The same resize with a size per frame: frame k (uint8 BGR at the top-left of slot k of slot_h x slot_w, e.g. the output of
 * sy_jpeg_decode_sized) of sizes[k] = (h, w, dst_h, dst_w) is resized h x w -> dst_h x dst_w (none when equal) with
 * sy_letterbox's arithmetic and placed top-left on a canvas of 114: the evaluation preproc of data_augment_flip.py:151-167
 * (dst = (int(h * r), int(w * r)), r = min(out_h / h, out_w / w)) or the driver's plain resize (dst = out) per stream.
 * With every row equal to (h, w, dst_h, dst_w) the output is sy_letterbox's.  A row that does not fit the slot or the canvas
 * leaves image k untouched. */
typedef struct SyLetterboxSizedDesc {
  const uint8_t* src;      /* [n][slot_h][slot_w][3] */
  int32_t n, slot_h, slot_w;
  const int32_t* sizes;    /* [n][4] device int32: h, w, dst_h, dst_w */
  int32_t out_h, out_w;
  float* out;              /* [n][3][out_h][out_w] */
} SyLetterboxSizedDesc;
int sy_letterbox_sized(const SyLetterboxSizedDesc* d, sy_stream_t stream);
/* The same resize into uint8 frames: frame k of sizes[k] = (h, w, dst_h, dst_w) at the top-left of slot k of src is
 * resized h x w -> dst_h x dst_w with sy_letterbox's arithmetic (cv2.resize INTER_LINEAR on uint8, bit for bit; a copy
 * when equal) into the top-left of slot k of out [n][out_h][out_w][3], channel order kept: mmcv.imrescale(img, s,
 * interpolation="bilinear") with dst = (int(h * s + 0.5), int(w * s + 0.5)).  The rest of each out slot is not written;
 * a row that does not fit the slots leaves out slot k untouched.  SY_EINVAL: a null pointer, src == out, or a side
 * outside 1..65535 or a slot of 2^31 bytes or more. */
typedef struct SyResizeSizedDesc {
  const uint8_t* src;      /* [n][slot_h][slot_w][3] */
  int32_t n, slot_h, slot_w;
  const int32_t* sizes;    /* [n][4] device int32: h, w, dst_h, dst_w */
  int32_t out_h, out_w;
  uint8_t* out;            /* [n][out_h][out_w][3] */
} SyResizeSizedDesc;
int sy_resize_sized(const SyResizeSizedDesc* d, sy_stream_t stream);

/* ---- Raw camera frames ----
 * YUV frames of camera streams of different sizes -> uint8 BGR frames at the top-left of slots of one size (the slots
 * sy_jpeg_decode_sized writes and sy_letterbox_sized reads), bit-identical to cv2.cvtColor with the code named beside each
 * format.  OpenCV's BT.601 limited-range fixed point: y = max(Y - 16, 0) * 1220542, u = U - 128, v = V - 128,
 * B = clip((y + 2116026 u + 2^19) >> 20), G = clip((y - 852492 v - 409993 u + 2^19) >> 20), R = clip((y + 1673527 v + 2^19)
 * >> 20); every pixel of a 2x2 (4:2:0) or 2x1 (4:2:2) group takes the group's chroma sample (replicated, not interpolated).
 * Frame i is the first h * w * 3 / 2 (4:2:0) or h * w * 2 (4:2:2) bytes of row i of src, laid out as cv2 takes it: */
enum {
  SY_YUV_NV12 = 0,   /* COLOR_YUV2BGR_NV12: Y plane [h][w], then interleaved U, V [h / 2][w / 2][2] */
  SY_YUV_NV21 = 1,   /* COLOR_YUV2BGR_NV21: Y plane, then interleaved V, U */
  SY_YUV_I420 = 2,   /* COLOR_YUV2BGR_I420: Y plane, U plane [h / 2][w / 2], V plane [h / 2][w / 2] */
  SY_YUV_YV12 = 3,   /* COLOR_YUV2BGR_YV12: Y plane, V plane, U plane */
  SY_YUV_YUY2 = 4,   /* COLOR_YUV2BGR_YUY2 (YUYV): [h][w / 2] groups Y0 U Y1 V */
  SY_YUV_UYVY = 5    /* COLOR_YUV2BGR_UYVY: [h][w / 2] groups U Y0 V Y1 */
};
/* sizes[i] = (h, w) of frame i.  A row with h = 0 means no frame this tick, and a row that is odd where the format
 * subsamples (4:2:0: h or w; 4:2:2: w), does not fit the slot, or whose frame is longer than max_bytes, also leaves slot i
 * untouched.  Reads no byte of row i past frame i's own bytes, only device memory; never synchronises (capturable). */
typedef struct SyYuvToBgrSizedDesc {
  const uint8_t* src;      /* [n][max_bytes] */
  int32_t n;
  int64_t max_bytes;       /* row pitch of src */
  const int32_t* sizes;    /* [n][2] device int32: h, w */
  int32_t format;          /* SY_YUV_* */
  int32_t slot_h, slot_w;
  uint8_t* out;            /* [n][slot_h][slot_w][3] BGR */
} SyYuvToBgrSizedDesc;
int sy_yuv_to_bgr_sized(const SyYuvToBgrSizedDesc* d, sy_stream_t stream);

/* 8-bit Bayer mosaics of camera streams of different sizes -> uint8 BGR frames at the top-left of the same slots,
 * bit-identical to cv2.cvtColor(raw, COLOR_Bayer<pattern>2BGR) (bilinear) or COLOR_Bayer<pattern>2BGR_EA (edge-aware).
 * Off the border (rows 1..h-2, columns 1..w-2) a pixel keeps its own colour; at a green site the colour of the left and
 * right neighbours is their mean (a + b + 1) >> 1 and that of the upper and lower neighbours theirs; at a red or blue
 * site the other of the two is the mean of the four diagonals (a + b + c + d + 2) >> 2 and green is the mean of the four
 * edge neighbours (bilinear) or, edge-aware, of the vertical pair where |left - right| > |up - down|, else of the
 * horizontal pair.  Column 0 copies column 1 and column w-1 column w-2, then row 0 copies row 1 and row h-1 row h-2.  A
 * frame of fewer than 3 rows or columns is black, as cv2 makes it.  Frame i is the first h * w bytes of row i of src,
 * row-major [h][w]; the pattern is the colour order of its top-left 2x2 (cv2's RGGB codes alias its BG ones): */
enum {
  SY_BAYER_RGGB = 0,   /* COLOR_BayerRGGB2BGR[_EA] = COLOR_BayerBG2BGR[_EA] */
  SY_BAYER_BGGR = 1,   /* COLOR_BayerBGGR2BGR[_EA] = COLOR_BayerRG2BGR[_EA] */
  SY_BAYER_GBRG = 2,   /* COLOR_BayerGBRG2BGR[_EA] = COLOR_BayerGR2BGR[_EA] */
  SY_BAYER_GRBG = 3    /* COLOR_BayerGRBG2BGR[_EA] = COLOR_BayerGB2BGR[_EA] */
};
enum {
  SY_DEMOSAIC_BILINEAR = 0,   /* COLOR_Bayer*2BGR */
  SY_DEMOSAIC_EA = 1          /* COLOR_Bayer*2BGR_EA (value 2 is kept for VNG, not built) */
};
/* sizes[i] = (h, w) of frame i.  A row with h = 0 means no frame this tick; a row that does not fit the slot, or whose
 * h * w is more than max_bytes, also leaves slot i untouched.  Nothing of slot i outside frame i's h x w is written.
 * Reads no byte of row i past frame i's own h * w, only device memory; never synchronises (capturable). */
typedef struct SyBayerToBgrSizedDesc {
  const uint8_t* src;      /* [n][max_bytes] */
  int32_t n;
  int64_t max_bytes;       /* row pitch of src */
  const int32_t* sizes;    /* [n][2] device int32: h, w */
  int32_t pattern;         /* SY_BAYER_* */
  int32_t algo;            /* SY_DEMOSAIC_* */
  int32_t slot_h, slot_w;
  uint8_t* out;            /* [n][slot_h][slot_w][3] BGR */
} SyBayerToBgrSizedDesc;
int sy_bayer_to_bgr_sized(const SyBayerToBgrSizedDesc* d, sy_stream_t stream);

/* ---- JPEG decode ----
 * Batched decode of the training frames' JPEG files into what cv2.imread(path) returns for them (uint8 BGR, bit-identical),
 * replacing the host decodes of exps/dataset/tal_flip_one_future_argoversedataset.py:195,216,
 * tal_flip_two_future_argoversedataset.py:207,228 and still_argoversedataset.py:160.  Reads only device memory and never
 * synchronises, so it can be captured in a CUDA graph in front of sy_letterbox.
 * Decoded streams: baseline (SOF0) or extended sequential (SOF1) 8-bit Huffman JPEG with three YCbCr components in one
 * interleaved scan, luma sampling 1x1, 2x1 or 2x2 (chroma 1x1), any Huffman tables, 8- or 16-bit quantisation tables, with
 * or without restart intervals, any size.  Everything else, and every damaged stream, gets a non-zero status[i] and image
 * i's output is left untouched; the other images of the batch decode as usual.  The decoder reads no input byte at or past
 * lengths[i] and writes nothing outside image i's output row.
 * Descriptor errors return SY_EINVAL; problems with the stream contents go only to status[]. */
enum {
  SY_JPEG_OK = 0,
  SY_JPEG_EHEADER = 1,       /* not a JPEG, malformed or truncated marker segments, undefined or invalid tables, or
                              * lengths[i] outside [4, max_bytes] */
  SY_JPEG_EUNSUPPORTED = 2,  /* progressive, arithmetic, lossless, hierarchical, 12-bit, not 3 components, RGB (Adobe
                              * transform 0), other sampling factors or more than one scan */
  SY_JPEG_EORIENTATION = 3,  /* an EXIF orientation other than 1 (cv2.imread would rotate the image) */
  SY_JPEG_ESIZE = 4,         /* the frame's size differs from the descriptor's h x w */
  SY_JPEG_EDATA = 5          /* corrupt or truncated entropy-coded data */
};
typedef struct SyJpegDecodeDesc {
  const uint8_t* bytes;     /* [n][max_bytes] file bytes, image i in the first lengths[i] bytes of row i */
  const int32_t* lengths;   /* [n] device int32 */
  int32_t n;
  int64_t max_bytes;        /* row pitch of bytes (1 .. 2^28) */
  int32_t h, w;             /* the size every image must have */
  uint8_t* out;             /* [n][h][w][3] BGR */
  int32_t* status;          /* [n] device int32, SY_JPEG_* */
  void* workspace;          /* sy_jpeg_decode_workspace_bytes(n, max_bytes, h, w) bytes, 256-byte aligned */
  size_t workspace_bytes;
} SyJpegDecodeDesc;
size_t sy_jpeg_decode_workspace_bytes(int32_t n, int64_t max_bytes, int32_t h, int32_t w);
int sy_jpeg_decode(const SyJpegDecodeDesc* d, sy_stream_t stream);
/* The same decoder with a size per image, for camera streams of different sizes (the frames cv2.imread gives the driver's
 * loop, sAP/streamyolo/streamyolo_det.py:176-181): image i must be sizes[i] = (h, w) with h <= max_h and w <= max_w, else
 * it gets SY_JPEG_ESIZE and is left untouched; it is written at the top-left of slot i of out [n][max_h][max_w][3] (row
 * pitch max_w * 3; the rest of the slot is not written).  The workspace is sized by the slot. */
typedef struct SyJpegDecodeSizedDesc {
  const uint8_t* bytes;     /* [n][max_bytes] file bytes, image i in the first lengths[i] bytes of row i */
  const int32_t* lengths;   /* [n] device int32 */
  int32_t n;
  int64_t max_bytes;        /* row pitch of bytes (1 .. 2^28) */
  const int32_t* sizes;     /* [n][2] device int32: the (h, w) image i must have */
  int32_t max_h, max_w;     /* slot size */
  uint8_t* out;             /* [n][max_h][max_w][3] BGR */
  int32_t* status;          /* [n] device int32, SY_JPEG_* */
  void* workspace;          /* sy_jpeg_decode_sized_workspace_bytes(n, max_bytes, max_h, max_w) bytes, 256-byte aligned */
  size_t workspace_bytes;
} SyJpegDecodeSizedDesc;
size_t sy_jpeg_decode_sized_workspace_bytes(int32_t n, int64_t max_bytes, int32_t max_h, int32_t max_w);
int sy_jpeg_decode_sized(const SyJpegDecodeSizedDesc* d, sy_stream_t stream);

/* ---- JPEG encode ----
 * Batched encode of uint8 BGR images of their own sizes into the bytes cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY,
 * quality]) returns for them, with cv2's other defaults (replacing the host cv2.imwrite of recorded camera frames):
 * baseline SOF0, YCbCr 4:2:0, libjpeg's quality-scaled Annex K tables, the standard Huffman tables, no restart interval,
 * JFIF 1.01 APP0 with density 1:1; segments SOI APP0 DQT DQT SOF0 DHT x 4 SOS, the scan, EOI.  Image i is sizes[i] =
 * (h, w) at the top-left of slot i of src [n][max_h][max_w][3] (the slots sy_jpeg_decode_sized and sy_yuv_to_bgr_sized
 * write); its file goes to the first lengths[i] bytes of row i of out.  Per image status: */
enum {
  SY_JPEG_ENCODE_OK = 0,
  SY_JPEG_ENCODE_EOVERFLOW = 1,   /* the file does not fit in max_bytes: lengths[i] = 0, nothing written past max_bytes */
  SY_JPEG_ENCODE_ESIZE = 2        /* sizes[i] has h or w below 1 or outside the slot: lengths[i] = 0, row i untouched */
};
/* The sizes are read on the device only, so a captured graph follows sizes written before each replay.  Never
 * synchronises (capturable).  SY_EINVAL: quality outside 1..100, a slot or max_bytes outside the limits of
 * sy_jpeg_encode_workspace_bytes, a null or misaligned pointer, or a short workspace. */
typedef struct SyJpegEncodeDesc {
  const uint8_t* src;       /* [n][max_h][max_w][3] BGR */
  const int32_t* sizes;     /* [n][2] device int32: h, w (4-byte aligned) */
  int32_t n;
  int32_t max_h, max_w;     /* slot size */
  int32_t quality;          /* 1..100 */
  uint8_t* out;             /* [n][max_bytes] */
  int64_t max_bytes;        /* row pitch of out (1 .. 2^31) */
  int64_t* lengths;         /* [n] device int64 (8-byte aligned): the file's length, 0 where status != OK */
  int32_t* status;          /* [n] device int32 (4-byte aligned), SY_JPEG_ENCODE_* */
  void* workspace;          /* sy_jpeg_encode_workspace_bytes(n, max_h, max_w, max_bytes) bytes, 256-byte aligned */
  size_t workspace_bytes;
} SyJpegEncodeDesc;
/* 0 for n outside 1..65535, a slot side outside 1..65535, max_bytes outside 1..2^31, or a slot of 2^32 / 1660 blocks or
 * more */
size_t sy_jpeg_encode_workspace_bytes(int32_t n, int32_t max_h, int32_t max_w, int64_t max_bytes);
/* A length no h x w file exceeds, whatever its content and quality: 623 header bytes, EOI, and every one of the
 * 6 * ceil(h / 16) * ceil(w / 16) blocks at 1660 bits (the longest DC code and its 11 bits, then 63 AC coefficients of
 * the longest AC code and 10 bits each), every scan byte followed by a stuffed 00.  0 for a side outside 1..65535. */
int64_t sy_jpeg_encode_max_bytes(int32_t h, int32_t w);
int sy_jpeg_encode(const SyJpegEncodeDesc* d, sy_stream_t stream);

/* ---- detection drawing (the sAP toolkit's visualisation) ----
 * sy_draw_boxes: the box branch of vis_obj_fancy (sAP/vis/vis_det_th.py:99-120, masks None, no text) on n uint8 images
 * of their own sizes: image i is sizes[i] = (h, w) at the top-left of slot i of src [n][max_h][max_w][3] and is drawn
 * into the same place of dst (dst == src draws in place).  With the first counts[i] boxes of row i (x1, y1, x2, y2,
 * already rounded; corners in either order) and their labels, in list order:
 *   1. fill (cv2.rectangle(img, ..., thickness=-1) then cv2.addWeighted(img_filled, 0.8, img, 0.2, 0), :101-110): a pixel
 *      in at least one box's [min(x1,x2), max(x1,x2)] x [min(y1,y2), max(y1,y2)] (inclusive) becomes
 *      rint(0.8f * v + 0.2f * p) per channel, p the palette colour of the last such box;
 *   2. contours (cv2.rectangle(img, ..., thickness=2), :112-120): a pixel within Chebyshev distance 1 of at least one
 *      box's border, except the four pixels diagonally outside its corners, becomes the palette colour of the last such
 *      box.
 * The palette is uint8 [P][3] in the images' channel order.  A box whose label is outside [0, P) is not drawn (the host
 * refuses those); counts are clamped to [0, K]; an image whose size row is below 1 or outside the slot is left alone.
 * Pixels outside an image and pixels no box touches are not written.  Boxes, labels, counts and sizes are read on the
 * device only, so a captured graph follows what is written before each replay; the result does not depend on thread
 * scheduling.  SY_EINVAL: a null pointer, n or a slot side outside 1..65535, K outside 1..2^24, P outside 1..65536, or a
 * dst slot shape other than src's. */
typedef struct SyDrawBoxesDesc {
  const uint8_t* src;       /* [n][max_h][max_w][3] */
  const int32_t* sizes;     /* [n][2] device int32: h, w */
  int32_t n;
  int32_t max_h, max_w;     /* src's slot size */
  const int32_t* boxes;     /* [n][K][4] x1, y1, x2, y2 */
  const int32_t* labels;    /* [n][K] */
  const int32_t* counts;    /* [n] */
  int32_t K;
  const uint8_t* palette;   /* [P][3] */
  int32_t P;
  uint8_t* dst;             /* [n][dst_h][dst_w][3], may be src */
  int32_t dst_h, dst_w;     /* must equal max_h, max_w */
} SyDrawBoxesDesc;
int sy_draw_boxes(const SyDrawBoxesDesc* d, sy_stream_t stream);

/* sy_vis_det_boxes: a streaming tick's NMS rows -> sy_draw_boxes's boxes, labels and counts, as the host path from the
 * driver's output to vis_obj_fancy computes them: the score obj * class_conf in fp32 (stream.sized_output), rows kept
 * where score >= score_th in fp32 (vis_det_th.py:81-83; -inf keeps every row, the script's score_th <= 0), in order; the
 * boxes through the ltrb -> ltwh -> ltrb round trip of streaming_eval.py and vis_det_th.py:232 (w = x2 - x1, then
 * x1 + w, in fp32) and rounded half to even (.round().astype(np.int32), :97; NaN, infinities and values outside int32
 * become INT_MIN, as that cast gives on x86-64); the label is class_pred.  det is
 * [S][A][7] (x1, y1, x2, y2, obj, class_conf, class_pred), stream s's first count[s] rows valid (clamped to [0, A]);
 * boxes [S][A][4], labels [S][A], counts [S] are written.  SY_EINVAL: a null pointer, S outside 1..65535 or A outside
 * 1..2^24. */
typedef struct SyVisDetBoxesDesc {
  const float* det;         /* [S][A][7] */
  const int32_t* count;     /* [S] */
  int32_t S, A;
  float score_th;
  int32_t* boxes;           /* [S][A][4] */
  int32_t* labels;          /* [S][A] */
  int32_t* counts;          /* [S] */
} SyVisDetBoxesDesc;
int sy_vis_det_boxes(const SyVisDetBoxesDesc* d, sy_stream_t stream);

/* sy_draw_outlines: the drawing of the sAP toolkit's vis_det (sAP/det/__init__.py:103-175, masks None) on n uint8
 * images of their own sizes, in place: image i is sizes[i] = (h, w) at the top-left of slot i of img [n][max_h][max_w][3].
 * Every pixel of
 *   - the first counts[i] boxes of row i (x1, y1, x2, y2, already rounded; corners in any order): the four 1-pixel lines
 *     cv2.rectangle(img, (x1, y1), (x2, y2), color, thickness=1) draws, [min x, max x] x {y1, y2} and
 *     {x1, x2} x [min y, max y], clipped to the image;
 *   - the first n_points[i] entries of row i of points: pixel y * w + x of image i (the host's cv2.putText strokes),
 *     entries outside [0, h * w) ignored;
 * becomes ``color`` (3 values in the images' channel order).  Every touched pixel gets the same colour, so the result is
 * the union of the touched pixels whatever the order of the writes.  Pixels outside an image and pixels nothing touches
 * are not written; counts and n_points are clamped to [0, K] and [0, M]; an image whose size row is below 1 or outside
 * the slot is left alone.  Sizes, boxes, counts, points and n_points are read on the device only, so a captured graph
 * follows what is written before each replay.  SY_EINVAL: a null pointer, n or a slot side outside 1..65535, a slot of
 * 2^31 pixels or more, K or M outside 1..2^24. */
typedef struct SyDrawOutlinesDesc {
  uint8_t* img;             /* [n][max_h][max_w][3], drawn in place */
  const int32_t* sizes;     /* [n][2] device int32: h, w */
  int32_t n;
  int32_t max_h, max_w;     /* slot size */
  const int32_t* boxes;     /* [n][K][4] x1, y1, x2, y2 */
  const int32_t* counts;    /* [n] */
  int32_t K;
  const int32_t* points;    /* [n][M] pixel indices y * w + x */
  const int32_t* n_points;  /* [n] */
  int32_t M;
  uint8_t color[3];
} SyDrawOutlinesDesc;
int sy_draw_outlines(const SyDrawOutlinesDesc* d, sy_stream_t stream);

/* sy_splice_frames: the split screen of the sAP toolkit's vis_contrast.py (sAP/vis/vis_contrast.py:148-165) on n pairs of
 * uint8 images of their own sizes, written into A in place: image i is sizes[i] = (h, w) at the top-left of slot i of a
 * and of b, both [n][max_h][max_w][3].  With splits[i] = (split, band_start, band_end) and c a pixel's coordinate along
 * the split axis (its column, or its row with horizontal = 1):
 *   band_start <= c < band_end   the band colour (:158-165, img[:, line_start:line_end] = line_color)
 *   otherwise c >= split         B's pixel (:148-156: B alone where split <= 0, img[:, split:] = img_B[:, split:])
 *   otherwise                    A's pixel, not written.
 * The host clamps split, band_start and band_end to [0, l] (l = w, or h with horizontal), an empty band being
 * band_start >= band_end; the kernel takes any int32 values as the rules above.  The colour is in the images' channel
 * order: (93, 159, 241) for BGR images is the script's RGB [241, 159, 93].  Pixels outside an image are not read or
 * written; an image whose size row is below 1 or outside the slot is left alone.  Sizes and splits are read on the device
 * only, so a captured graph follows what is written before each replay.  One launch, no synchronisation.  SY_EINVAL: a
 * null pointer, a == b, n or a slot side outside 1..65535, or horizontal other than 0 or 1. */
typedef struct SySpliceFramesDesc {
  uint8_t* a;               /* [n][max_h][max_w][3], written in place */
  const uint8_t* b;         /* [n][max_h][max_w][3] */
  const int32_t* sizes;     /* [n][2] device int32: h, w */
  const int32_t* splits;    /* [n][3] device int32: split, band_start, band_end */
  int32_t n;
  int32_t max_h, max_w;     /* slot size of a and b */
  int32_t horizontal;       /* 0: split along x (columns, the script's default), 1: along y (--horizontal) */
  uint8_t color[3];         /* the band colour */
} SySpliceFramesDesc;
int sy_splice_frames(const SySpliceFramesDesc* d, sy_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* STREAMYOLO_SM100_H_ */
