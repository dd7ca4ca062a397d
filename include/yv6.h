/* yv6.h -- C ABI of libyolov6_b200.so: the sm_90a kernels under the YOLOv6 hot path.
 *
 * The reference (meituan/YOLOv6 @ e86a483) has no native boundary: its hot path is PyTorch ops
 * behind a Python API.  This library sits *under* that API (SURVEY.md section 8b): the host side in
 * `yolov6_b200/` keeps the reference's Python signatures and calls these entry points through
 * ctypes with raw device pointers.  Every entry point
 *   - is `extern "C"`, takes plain pointers / sizes / a `cudaStream_t` passed as `void*`,
 *   - is asynchronous on that stream and allocates nothing the caller has to free,
 *   - returns 0 on success or a negative YV6_ERR_* code; `yv6_last_error()` then holds the message
 *     (the Python side raises RuntimeError, matching the reference's failure contract,
 *     yolov6/models/losses/loss.py:105 `except RuntimeError`).
 *
 * Layout conventions: activations are NHWC (channels innermost), bf16 unless stated; weights are
 * KRSC = [Cout][kh][kw][Cin] bf16; all strides are in ELEMENTS of the tensor's dtype.
 */
#ifndef YV6_H_
#define YV6_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YV6_ABI_VERSION 4

enum {
  YV6_OK = 0,
  YV6_ERR_ARG = -1,     /* invalid argument / unsupported shape */
  YV6_ERR_CUDA = -2,    /* a CUDA runtime / driver call failed */
  YV6_ERR_STATE = -3    /* handle not usable (wrong device, destroyed, ...) */
};

/* HARDSWISH = x * min(max(x + 3, 0), 6) / 6 (nn.Hardswish), HARDSIGMOID = min(max(x + 3, 0), 6) / 6 (nn.Hardsigmoid) */
enum { YV6_ACT_NONE = 0, YV6_ACT_RELU = 1, YV6_ACT_SILU = 2, YV6_ACT_SIGMOID = 3, YV6_ACT_HARDSWISH = 4, YV6_ACT_HARDSIGMOID = 5 };
enum { YV6_DT_BF16 = 0, YV6_DT_F32 = 1, YV6_DT_U8 = 2, YV6_DT_F16 = 3 };
#define YV6_PAD_SAME (-1000000)

typedef struct yv6_handle yv6_handle;

/* Per-device context: SM count, driver entry points (cuTensorMapEncodeTiled), scratch space. */
int yv6_create(int device, yv6_handle** out);
int yv6_destroy(yv6_handle* h);
/* Thread-local message of the last failing call on this thread. */
const char* yv6_last_error(void);
int yv6_abi_version(void);

/* ------------------------------------------------------------------------------------------------
 * Fused convolution: y = act(conv(x, w) + bias) [+ alpha * residual]
 *
 * Replaces, in deploy form, ConvModule.forward_fuse (yolov6/layers/common.py:50-54),
 * RepVGGBlock.forward with `rbr_reparam` (common.py:247-248), BottleRep's `+ alpha*x`
 * (common.py:605-608), the 1x1 convs of BiFusion / BepC3 / (CSP)SPPF (common.py:699-718,
 * 639-650, 140-158), the head stems / cls_preds / reg_preds incl. the sigmoid of
 * effidehead.py:85,112, and -- through y_*_stride/offset -- `torch.cat` of the necks
 * (reppan.py:228,232) and ConvTranspose2d k2 s2 (common.py:181-194, four 1x1 launches that
 * scatter to the 2x2 sub-grid).
 *
 * Implicit GEMM on wgmma: M = output pixels (tile = BWxBHxBI box, <=128 rows), N = Cout,
 * K = kh*kw*Cin.  A tiles are TMA box loads of the NHWC input shifted per filter tap (zero fill
 * out of bounds = padding; elementStrides = conv stride), B tiles are TMA loads of the KRSC
 * weights, accumulators live in registers, epilogue fuses bias/activation/residual/dtype/slice.
 *
 * nsplit = 1: bf16 operands, fp32 accumulate.
 * nsplit = 3: "bf16x3" fp32-equivalent mode -- x, w and y are three bf16 planes (hi, mid, lo) whose
 *             sum is the fp32 value; six plane-pair products are accumulated in fp32.
 * reserved0 = YV6_DT_F16 (operand dtype; 0 = bf16): x, w and res are fp16 and y is fp16 (y_dtype = YV6_DT_F16) or fp32;
 *             fp16 wgmma with fp32 accumulation, nsplit must be 1.  Outputs beyond fp16's range (65504) become +-inf.
 *             The tile plan is the one the bf16 operands get.
 * ---------------------------------------------------------------------------------------------- */
typedef struct yv6_conv_desc {
  /* input */
  const void* x;            /* bf16, pixel (n,h,w) channel c at ((n*H+h)*W+w)*x_c_total + c     */
  int32_t N, H, W, Cin;     /* Cin % 16 == 0                                                    */
  int32_t x_c_total;        /* channel pitch of the buffer x lives in (>= Cin, % 8 == 0)        */
  int64_t x_plane_stride;   /* elements between bf16x3 planes (ignored when nsplit == 1)        */
  /* weights / bias */
  const void* w;            /* bf16 KRSC [Cout][kh][kw][Cin]                                    */
  int64_t w_plane_stride;   /* elements between weight planes (nsplit == 3)                     */
  const float* bias;        /* fp32, length >= round_up(Cout, 256) (zero padded), or NULL       */
  int32_t Cout, kh, kw, stride, pad;
  int32_t act;              /* YV6_ACT_*                                                        */
  /* output: element (n,ho,wo,co) at y + n*y_img_stride + ho*y_h_stride + wo*y_w_stride + co   */
  void* y;
  int32_t y_dtype;          /* YV6_DT_BF16 or YV6_DT_F32                                        */
  int64_t y_img_stride, y_h_stride, y_w_stride;
  int64_t y_plane_stride;   /* nsplit == 3 and bf16 output only                                 */
  /* optional residual (bf16, same dtype/planes as x): y += alpha * res[...]                   */
  const void* res;
  float alpha;
  int64_t res_img_stride, res_h_stride, res_w_stride, res_plane_stride;
  int32_t nsplit;           /* 1 or 3                                                           */
  /* tuning overrides, 0 = auto */
  int32_t force_bw, force_bh, force_bi, force_bn, force_stages, force_grid;
  int32_t force_direct;     /* ignored: the epilogue always stores through the staged fp32 tile (field kept for the layout) */
  int32_t force_halo;       /* 3x3 s1 halo-reuse mainloop: 0 = auto, 1 = force on (if eligible), -1 = off */
  /* generalisations used by the backward pass (dgrad of stride-2 convs = four parity sub-convolutions with
   * 1- or 2-tap kernels): kh, kw in 1..3 independently; `pad` pads rows, pad_w columns (YV6_PAD_SAME = pad);
   * out_h / out_w > 0 override the output size (far-side reads are zero filled). */
  int32_t pad_w, out_h, out_w;
  int32_t force_groups;     /* ignored (field kept for the layout) */
  void* trace;              /* ignored (field kept for the layout) */
  /* ABI 2: column stride when it differs from the row stride (0 = `stride`).  A 3x3 stride-2 conv over few channels runs
   * faster on the "column-pair" view of its input -- [N, H, W/2, 2*Cin], a pure reinterpretation of NHWC memory -- as a
   * 3x2 kernel with stride (2, 1), pad_w = 1, out_w = W/2: the A rows become contiguous 2*Cin-channel pixels instead of
   * every other Cin-channel pixel (see yolov6_b200/engine.py). */
  int32_t stride_w;
  int32_t force_pair;       /* CTA pairs (clusters of two CTAs on adjacent M tiles, each loading half of the weight tile and
                             * multicasting it into both): 1 = on whenever the layer has >= 2 M tiles; 0 (auto) and -1 = off. */
  /* ABI 4.  pair_view = 1: this 3x2 / stride (2, 1) descriptor is the column-pair view of a 3x3 stride-2 conv (see stride_w) and
   * its weights are zero where the view has no tap -- w[:, :, 0, 0 .. Cin/2) (left tap, even pixel of the pair).  The halo-reuse
   * mainloop (one 9 x 33 input box per 8 x 16 output tile instead of one box per tap) then skips the all-zero 64-channel
   * blocks, so the view costs no extra MACs when Cin/2 % 64 == 0.  0 = no promise (every block is multiplied). */
  int32_t pair_view;
  int32_t reserved0;        /* operand dtype: 0 = bf16, YV6_DT_F16 = fp16 (see above); anything else is YV6_ERR_ARG */
} yv6_conv_desc;

int yv6_conv_fwd(yv6_handle* h, const yv6_conv_desc* d, void* stream);
/* Reports the tile plan yv6_conv_fwd would use: out[0..9] = BW,BH,BI,BN,KB,stages,grid,tiles,halo,
 * (A stages * 100 + B resident). */
int yv6_conv_plan(yv6_handle* h, const yv6_conv_desc* d, int32_t* out10);
/* Host-only twin: the plan for a device with the stated properties (H100 SXM: 132 SMs, 232448 bytes of opt-in shared memory,
 * 66 co-resident 2-CTA clusters), no CUDA call -- the tile planner can be exercised where there is no GPU (tests/test_conv_planner.py).
 * out[0..9] as above, out[10] = dynamic shared memory in bytes (fails if it exceeds the device), out[11] = threads per CTA. */
int yv6_conv_plan_host(int num_sms, int max_smem_optin, int max_clusters, const yv6_conv_desc* d, int32_t* out12);

/* ------------------------------------------------------------------------------------------------
 * Stem: first 3x3 stride-2 conv on the 3-channel NCHW image, deploy form of `backbone.stem`
 * (reference yolov6/models/efficientrep.py:28-33), fused with the input conversion of
 * Trainer.prepro_data / Inferer.process_image (core/engine.py:407-410, core/inferer.py:162-171):
 * x is NCHW fp32 in [0,1] or NCHW uint8 (then scaled by in_scale = 1/255 on the fly).
 * Output NHWC bf16 (1 or 3 planes).  w / bias are DEVICE pointers: w is fp32 [3][3][3][Cout]
 * (tap-major, Cout innermost), bias fp32 [Cout] or NULL.
 * ---------------------------------------------------------------------------------------------- */
typedef struct yv6_stem_desc {
  const void* x;            /* device, [N,3,H,W] fp32 or uint8                                  */
  int32_t x_dtype;          /* YV6_DT_F32 or YV6_DT_U8                                          */
  float in_scale;           /* multiplier for uint8 input (1/255)                               */
  int32_t N, H, W;
  const float* w;           /* device fp32 [kh=3][kw=3][cin=3][Cout]                            */
  const float* bias;        /* device fp32 [Cout] or NULL                                       */
  int32_t Cout, act;        /* Cout in {16,32,48,64}                                            */
  void* y;                  /* device bf16 [planes][N,H/2,W/2,Cout]                             */
  int64_t y_plane_stride;
  int32_t nsplit;           /* 1 or 3                                                           */
  int32_t fp32_math;        /* nsplit == 1 only: 1 = fp32 image / weights on CUDA cores (training), 0 = bf16
                               image / weights on tensor cores (inference)                          */
  int32_t force_sync_loads; /* ABI 3, tuning: 1 = register-prefetch kernel even where the cp.async ring variant applies
                               (fp32 images with 16-byte aligned rows) */
} yv6_stem_desc;
int yv6_stem_fwd(yv6_handle* h, const yv6_stem_desc* d, void* stream);
/* The same with fp16 output (one plane, tensor cores: fp16 image / weights, fp32 accumulate; nsplit = 1, fp32_math = 0). */
int yv6_stem_fwd_f16(yv6_handle* h, const yv6_stem_desc* d, void* stream);

/* SPPF / CSPSPPF pooling (reference yolov6/layers/common.py:106-112,150-158): buf is the 4C-wide
 * NHWC concat buffer whose channel slice [0,C) holds x; writes the 5x5 / 9x9 / 13x13 clipped-window
 * maxima (= three chained MaxPool2d(5,1,2)) into slices [C,2C), [2C,3C), [3C,4C). */
int yv6_sppf_pool(yv6_handle* h, void* buf, int32_t N, int32_t H, int32_t W, int32_t C, int32_t c_total,
                  int32_t nsplit, int64_t plane_stride, void* stream);
/* The same on an fp16 buffer (nsplit = 1, C % 16 == 0). */
int yv6_sppf_pool_f16(yv6_handle* h, void* buf, int32_t N, int32_t H, int32_t W, int32_t C, int32_t c_total,
                      int32_t nsplit, int64_t plane_stride, void* stream);

/* ------------------------------------------------------------------------------------------------
 * YOLOv6Lite (reference yolov6/models/yolo_lite.py; layers/common.py:740-934): the layers that are not dense convolutions.
 * The 1x1 ConvBNHS convs run on yv6_conv_fwd with act = YV6_ACT_HARDSWISH, `conv_0` on yv6_stem_fwd.
 * Activations are NHWC bf16 channel slices: x / y point at the slice's first channel, *_c_total / *_pitch is the channel
 * pitch of the buffer; nsplit = 3: three bf16 planes *_plane_stride elements apart, computed on as their fp32 sum.
 *
 * yv6_dwconv_fwd: depthwise conv (groups = C), k in {3, 5}, stride 1 or 2, padding k / 2, output ((H-1)/s+1) x ((W-1)/s+1);
 *   y = act(conv(x, w) + bias), act NONE or HARDSWISH.  w fp32 [k*k][C] (tap-major, channel innermost), bias fp32 [C] or NULL.
 *   Any C and slice offset; channels of y outside the slice are not written.
 * yv6_dwconv_fwd_f16: the same on fp16 activations (nsplit = 1); the weights stay fp32.
 * yv6_se_fwd: SEBlock in place on x: s = hardsigmoid(W2 relu(W1 mean_hw(x) + b1) + b2), x *= s per (image, channel).
 *   w1 fp32 [Cr][C], b1 [Cr], w2 [C][Cr], b2 [C]; C <= 512, Cr <= 128.  Deterministic: fixed summation order, no atomics.
 *   reserved0 = operand dtype: 0 = bf16, YV6_DT_F16 = fp16 x (nsplit = 1); anything else is YV6_ERR_ARG.
 * yv6_channel_shuffle: channel_shuffle(cat(a, b), 2) of two C-channel slices: y[.., 2j] = a[.., j], y[.., 2j+1] = b[.., j].
 * yv6_upsample2x: nearest 2x upsample of an [N, H, W, C] slice into a [N, 2H, 2W, .] slice.
 *   Both copy 16-bit elements bit for bit, so they serve fp16 activations as they are.
 * ---------------------------------------------------------------------------------------------- */
typedef struct yv6_dw_desc {
  const void* x;
  int32_t N, H, W, C;
  int32_t x_c_total, y_c_total;
  int64_t x_plane_stride, y_plane_stride;
  const float* w;
  const float* bias;
  int32_t k, stride, act, nsplit;
  void* y;
} yv6_dw_desc;
int yv6_dwconv_fwd(yv6_handle* h, const yv6_dw_desc* d, void* stream);
int yv6_dwconv_fwd_f16(yv6_handle* h, const yv6_dw_desc* d, void* stream);

typedef struct yv6_se_desc {
  void* x;
  int32_t N, HW, C, Cr;
  int64_t c_total, plane_stride;
  const float* w1;
  const float* b1;
  const float* w2;
  const float* b2;
  int32_t nsplit, reserved0;   /* reserved0: operand dtype (0 = bf16, YV6_DT_F16) */
} yv6_se_desc;
int yv6_se_fwd(yv6_handle* h, const yv6_se_desc* d, void* stream);

int yv6_channel_shuffle(yv6_handle* h, const void* a, int64_t a_pitch, int64_t a_plane, const void* b, int64_t b_pitch,
                        int64_t b_plane, int64_t pixels, int32_t C, void* y, int64_t y_pitch, int64_t y_plane, int32_t nsplit,
                        void* stream);
int yv6_upsample2x(yv6_handle* h, const void* x, int64_t x_pitch, int64_t x_plane, int32_t N, int32_t H, int32_t W, int32_t C,
                   void* y, int64_t y_pitch, int64_t y_plane, int32_t nsplit, void* stream);

/* Eval-mode head decode (reference yolov6/models/effidehead.py:106-139, assigners/anchor_generator.py
 * :13-33, utils/general.py:32-43): cls [B,A,nc] fp32 (post-sigmoid), reg [B,A,reg_ch] fp32 (ltrb, or
 * 4*(reg_max+1) DFL logits) -> out [B,A,5+nc] = (cx,cy,w,h in pixels, 1, cls).  Levels are given by
 * their grid sizes and strides; A = sum(lvl_h*lvl_w). */
int yv6_head_decode(yv6_handle* h, const float* cls, const float* reg, float* out, int32_t B, int32_t nc,
                    int32_t reg_ch, int32_t nl, const int32_t* lvl_h, const int32_t* lvl_w,
                    const float* lvl_stride, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Batched NMS: reference yolov6/utils/nms.py:31-105 (`non_max_suppression`) including the greedy
 * suppression of torchvision.ops.nms (nms.py:96), for ALL images in one call.
 *   pred [B,A,5+nc] fp32 (xywh, obj, cls).  Candidate rule, class-offset boxes (+cls*4096), stable
 *   descending order, float-IoU-vs-double-threshold comparison and max_nms = 30000 truncation follow
 *   the reference's CPU path bit for bit (fp32 ops issued without FMA contraction).
 *   class_mask: NULL or nc bytes (1 = keep class) -- the `classes` filter.
 * Outputs: out [B,max_det,6] (xyxy, conf, cls), out_count [B], out_src [B,max_det,2] (anchor, class).
 * workspace: device scratch of at least yv6_nms_workspace_bytes(B, A, nc, multi_label) bytes.
 * overflow (device int32, may be NULL) is set to 1 if an image produced more candidates than the
 * workspace holds (only possible with multi_label and > 65536 (anchor, class) pairs above conf).
 * ---------------------------------------------------------------------------------------------- */
int64_t yv6_nms_workspace_bytes(int32_t B, int32_t A, int32_t nc, int32_t multi_label);
int yv6_nms_batched(yv6_handle* h, const float* pred, int32_t B, int32_t A, int32_t nc, float conf_thres,
                    double iou_thres, int32_t agnostic, int32_t multi_label, const uint8_t* class_mask,
                    int32_t max_det, float* out, int32_t* out_count, int32_t* out_src, int32_t* overflow,
                    void* workspace, int64_t workspace_bytes, void* stream);

/* Same NMS on the head tensors, without materialising `pred`: cls [B,A,nc] (post-sigmoid) and reg [B,A,reg_ch] as the prediction
 * convs write them, levels as for yv6_head_decode.  Candidate boxes are decoded on demand with the operation order of
 * yv6_head_decode, so the kept rows are bit-identical to yv6_head_decode + yv6_nms_batched (objectness is 1, effidehead.py:133-138). */
int yv6_nms_batched_head(yv6_handle* h, const float* cls, const float* reg, int32_t B, int32_t nc, int32_t reg_ch, int32_t nl,
                         const int32_t* lvl_h, const int32_t* lvl_w, const float* lvl_stride, float conf_thres, double iou_thres,
                         int32_t agnostic, int32_t multi_label, const uint8_t* class_mask, int32_t max_det, float* out,
                         int32_t* out_count, int32_t* out_src, int32_t* overflow, void* workspace, int64_t workspace_bytes,
                         void* stream);

/* Evaluation post-processing of the batched NMS output (SURVEY.md 8f N4): Evaler.scale_coords + box_convert + the top-left
 * shift of Evaler.convert_to_coco_format (yolov6/core/evaler.py:333-373) for all images in one launch.
 * det [B,max_det,6] (xyxy, conf, cls) and count [B] as written by yv6_nms_batched; meta [B,6] fp32 = (gain_h, gain_w, pad_x,
 * pad_y, h0, w0) per image; out [B,max_det,6] = (x_topleft, y_topleft, w, h, conf, cls) in original-image pixels, rows
 * beyond count[b] zeroed.  fp32 operation order of the reference (identical decimal output). */
int yv6_eval_boxes(yv6_handle* h, const float* det, const int32_t* count, const float* meta, int32_t B, int32_t max_det,
                   float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Precision / recall metric of the Evaler (do_pr_metric, core/evaler.py:109-226; utils/metrics.py:13-215) over a dataset.
 * The accumulators live in device buffers the caller owns, described by yv6_pr_state; the caller zeroes nt, npred,
 * matrix and flags before the first image.  Slot s = image * max_det + row of conf / cls / correct.
 *
 * yv6_pr_match: one launch per batch, images first_image .. first_image + B - 1 of the dataset.  det [B,max_det,6] / count
 *   [B] as yv6_nms_batched writes them (max_det <= state max_det); targets [n_targets,6] fp32 (image in the batch, cls, x, y,
 *   w, h normalised), any row order; meta [B,6] as for yv6_eval_boxes; H, W the letterboxed canvas; iouv [10] fp32 device
 *   table (torch.linspace(0.5, 0.95, 10)).  Writes each row's conf, cls and correct bits (bit t: correct at iouv[t], the
 *   rule of metrics.process_batch), ndet[image], adds label and prediction counts per class and, with confusion != 0,
 *   ConfusionMatrix.process_batch to matrix[pred][true] ((nc+1) x (nc+1), row / column nc = background).  flags[0] gets
 *   error bits (1: label class outside [0, nc) or not whole, 2: same for a detection, 4: an image has more labels than
 *   fit in shared memory), flags[1] = 1 once any row is correct.
 * yv6_pr_metric: ap_per_class + compute_ap + the Evaler's summary over images 0 .. n_images - 1, in float64.  px [1000]
 *   and x101 [101] are np.linspace(0, 1, 1000) / np.linspace(0, 1, 101) (device).  out (device, YV6_PR_OUT_SIZE(nc)
 *   doubles): p [nc][1000], r [nc][1000], f1 [nc][1000], ap [nc][10] (rows of classes without labels stay 0), nt [nc],
 *   matrix [(nc+1)^2] (0 without confusion), then map50, map, mp, mr, i* (last arg-max of f1.mean(0)), ok (0: no row is
 *   correct at any threshold -- map50 = map = mp = mr = 0 and i* = -1), flags[0], number of classes with labels.
 * ---------------------------------------------------------------------------------------------- */
typedef struct yv6_pr_state {
  int32_t max_images, max_det, nc, confusion;
  float* conf; float* cls;                              /* [max_images][max_det]                                          */
  uint16_t* correct;                                    /* [max_images][max_det]                                          */
  int32_t* ndet;                                        /* [max_images] rows per image                                     */
  int32_t* nt; int32_t* npred;                          /* [nc] labels / predictions per class                            */
  int32_t* matrix;                                      /* [(nc+1)*(nc+1)], may be NULL when confusion == 0               */
  int32_t* flags;                                       /* [2]                                                            */
} yv6_pr_state;
#define YV6_PR_OUT_SIZE(nc) ((int64_t)(nc) * 3010 + (int64_t)(nc) + ((int64_t)(nc) + 1) * ((int64_t)(nc) + 1) + 8)
int64_t yv6_pr_workspace_bytes(int32_t max_images, int32_t max_det);
int yv6_pr_match(yv6_handle* h, const yv6_pr_state* st, const float* det, const int32_t* count, int32_t B, int32_t max_det,
                 const float* targets, int32_t n_targets, const float* meta, int32_t H, int32_t W, const float* iouv,
                 int32_t first_image, void* stream);
int yv6_pr_metric(yv6_handle* h, const yv6_pr_state* st, int32_t n_images, const double* px, const double* x101, void* workspace,
                  int64_t workspace_bytes, double* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * COCO box mAP (pycocotools COCOeval, iouType 'bbox', default Params) over a dataset, in float64, as the reference's
 * Evaler.eval_model computes it (core/evaler.py:231-321).  Images are slots 0 .. n_images - 1 in np.unique(imgIds) order,
 * categories 0 .. n_cats - 1 the sorted gt category ids.  The caller owns every buffer: the gt table (uploaded once) and
 * the per-(slot, row) accumulators; it zeroes ndet and flags before the first image.  Area ranges, IoU and recall
 * thresholds are Params' float64 values, copied to the device by the caller.
 *
 * yv6_coco_update: one launch per batch on the batched NMS tensors.  det [B,max_det,6] / count [B] as yv6_nms_batched writes
 *   them, meta [B,6] as for yv6_eval_boxes, cls_cat [n_cls] int32 (class -> category index, -1: not a gt category),
 *   slots [B] int32 (-1: image not evaluated).  Each row becomes the detection pycocotools reads back from the Evaler's
 *   predictions.json: yv6_eval_boxes' box, then x_r = rint(x * 1e3) / 1e3 and s_r = rint(conf * 1e5) / 1e5 in double
 *   (round(v, 3) / round(v, 5) and a json round trip), area = w_r * h_r.
 * yv6_coco_load: the same for result rows given as doubles: rows [n][6] = (x, y, w, h, score, category index), grouped by
 *   image in result order, image b owning rows row_off[b] .. row_off[b+1] - 1 (at most state max_det).
 * Both then match per (image, category): stable sort by descending score, the first 100 kept, bbIou against the pair's gts
 *   and the greedy match of evaluateImg for every (area range, IoU threshold); bit a * 10 + t of tp / fp holds the
 *   outcome, rank the detection's place in its pair (255: beyond the 100 kept).  flags[0] bit 1: a detection class
 *   outside [0, n_cls) or not whole.
 * yv6_coco_accumulate: COCOeval.accumulate over every slot: precision and scores [10][101][n_cats][4][3], recall
 *   [10][n_cats][4][3] (device float64), -1 where pycocotools leaves -1.
 * ---------------------------------------------------------------------------------------------- */
typedef struct yv6_coco_state {
  int32_t n_images, n_cats, max_det, max_gts;           /* max_gts: the most gts of one (image, category)                 */
  const int32_t* gt_off;                                /* [n_images * n_cats + 1] CSR by (slot, category), file order   */
  const double* gt_box;                                 /* [G][4] x, y, w, h                                              */
  const double* gt_area;                                /* [G] the annotation's area field                                */
  const uint8_t* gt_flags;                              /* [G] bit 0: iscrowd, bit 1: id != 0                             */
  const int32_t* npig;                                  /* [n_cats][4] gts that are not ignored, per area range           */
  const double* area_rng;                               /* [4][2]                                                         */
  const double* iou_thrs;                               /* [10]                                                           */
  const double* rec_thrs;                               /* [101]                                                          */
  double* score;                                        /* [n_images][max_det] s_r                                        */
  int32_t* cat;                                         /* [n_images][max_det] category index, -1: dropped                */
  uint8_t* rank;                                        /* [n_images][max_det]                                            */
  uint64_t* tp; uint64_t* fp;                           /* [n_images][max_det]                                            */
  int32_t* ndet;                                        /* [n_images] rows stored                                         */
  int32_t* flags;                                       /* [1]                                                            */
} yv6_coco_state;
int64_t yv6_coco_workspace_bytes(int32_t n_images, int32_t max_det, int32_t n_cats);
int yv6_coco_update(yv6_handle* h, const yv6_coco_state* st, const float* det, const int32_t* count, const float* meta,
                    const int32_t* cls_cat, int32_t n_cls, const int32_t* slots, int32_t B, int32_t max_det, void* stream);
int yv6_coco_load(yv6_handle* h, const yv6_coco_state* st, const double* rows, const int32_t* row_off, const int32_t* slots, int32_t B,
                  void* stream);
int yv6_coco_accumulate(yv6_handle* h, const yv6_coco_state* st, void* workspace, int64_t workspace_bytes, double* precision,
                        double* recall, double* scores, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Serving from decoded frames: the two steps of the reference's Inferer around the model, for a whole batch per launch.
 * Per-image geometry table geo [B][YV6_LB_GEO] int32 (device) = (src_off, h0, w0, nh, nw, top, left, 0):
 *   src_off   byte offset of the image in `src` (images packed back to back, each uint8 HWC BGR [h0][w0][3]);
 *   nh, nw    new_unpad of letterbox (data_augment.py:43), top / left its integer border (:54-55), computed by the caller
 *             with the reference's Python expressions; the kernels recompute none of them.
 *
 * yv6_letterbox: letterbox(im, (H, W), auto=False) (data_augment.py:29-58) + HWC->CHW + BGR->RGB of Inferer.process_image
 *   (core/inferer.py:161-171) -> dst uint8 NCHW [B,3,H,W] (the stem's YV6_DT_U8 input; the 1/255 stays in the stem).
 *   Canvas outside [top, top+nh) x [left, left+nw) = 114; inside, cv2.resize INTER_LINEAR of the uint8 source, bit-exact,
 *   or a plain copy when (nh, nw) == (h0, w0).  A slot with nh = 0 is all border.  W % 16 == 0, dst 16-byte aligned.
 * yv6_letterbox_frames: the same canvases, but image b is read through srcs[b] (device [B] yv6_lb_src) instead of
 *   src + src_off, so each image may lie anywhere in device memory (a decoder's output, a crop view of a larger frame, a
 *   staging buffer) in either layout below; geo supplies everything else and its src_off is ignored.  The layout is data,
 *   so one captured graph serves any mix of layouts and frame locations.  Pitches are in bytes:
 *     YV6_LB_BGR_HWC  pixel (y, x) channel c (B, G, R) at base + y * row_pitch + x * 3 + c; plane_pitch unused (cv2 imread);
 *     YV6_LB_RGB_CHW  pixel (y, x) channel c (R, G, B) at base + c * plane_pitch + y * row_pitch + x (torchvision decoders).
 *   Canvas plane c reads source channel 2 - c of BGR HWC and source plane c of RGB CHW, so both give the canvas yv6_letterbox
 *   gives for the equivalent BGR HWC image.  A slot with nh = 0 reads nothing (its record may hold a null base).
 * yv6_rescale_boxes: Inferer.rescale((H, W), det[:, :4], (h0, w0)) followed by .round() (inferer.py:103, 173-188) on the
 *   NMS output det [B,max_det,6] / count [B] -> out [B,max_det,6] (x1, y1, x2, y2 in source pixels, conf, cls), rows
 *   beyond count[b] zeroed.  Reads h0, w0 of geo.  Ratio and padding are the reference's doubles, box math its fp32.
 * ---------------------------------------------------------------------------------------------- */
#define YV6_LB_GEO 8
enum { YV6_LB_BGR_HWC = 0, YV6_LB_RGB_CHW = 1 };
typedef struct {
  const uint8_t* base;         /* pixel (0, 0) of the image's first channel                                   */
  int64_t row_pitch;           /* bytes from one image row to the next                                        */
  int64_t plane_pitch;         /* bytes from one channel plane to the next (YV6_LB_RGB_CHW)                   */
  int32_t layout;              /* YV6_LB_BGR_HWC or YV6_LB_RGB_CHW                                            */
  int32_t reserved0;
} yv6_lb_src;
int yv6_letterbox(yv6_handle* h, const uint8_t* src, const int32_t* geo, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                  void* stream);
int yv6_letterbox_frames(yv6_handle* h, const yv6_lb_src* srcs, const int32_t* geo, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                         void* stream);
int yv6_rescale_boxes(yv6_handle* h, const float* det, const int32_t* count, const int32_t* geo, int32_t B, int32_t max_det,
                      int32_t H, int32_t W, float* out, void* stream);

/* yv6_letterbox_val: the Evaler's validation images, TrainValDataset.__getitem__ with augment=False
 *   (yolov6/data/datasets.py:189-198, 281-296): load_image's resize of the source to (nh, nw), then letterbox onto the batch
 *   canvas with scaleup=False -- which, the canvas being at least nh x nw, only pads -- + HWC->CHW + BGR->RGB, into dst
 *   uint8 NCHW [B,3,H,W].  Sources as for yv6_letterbox_frames (srcs, layouts, pitches); geo as above, with geo[7] the
 *   image's mode, chosen by the caller the way cv::resize chooses its path:
 *     YV6_VAL_COPY       (nh, nw) == (h0, w0): load_image's ratio is 1, the image is copied;
 *     YV6_VAL_LINEAR     cv2.INTER_LINEAR enlargement (ratio > 1), as yv6_letterbox;
 *     YV6_VAL_AREA       cv2.INTER_AREA shrink (ratio < 1), OpenCV's generic resizeArea_ path, bit-exact;
 *     YV6_VAL_AREA_FAST  cv2.INTER_AREA shrink whose scales h0 / nh and w0 / nw are both integers (resizeAreaFast_), bit-exact.
 *   Canvas outside [top, top+nh) x [left, left+nw) = 114; a slot with nh = 0 is all border and reads nothing.  The caller
 *   guarantees top + nh <= H and left + nw <= W.  W % 16 == 0, dst 16-byte aligned. */
enum { YV6_VAL_COPY = 0, YV6_VAL_LINEAR = 1, YV6_VAL_AREA = 2, YV6_VAL_AREA_FAST = 3 };
int yv6_letterbox_val(yv6_handle* h, const yv6_lb_src* srcs, const int32_t* geo, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                      void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training augmentation from decoded frames: TrainValDataset.__getitem__ (yolov6/data/datasets.py:166-255) with
 * augment=True for a whole batch, bit-exact against the cv2 calls it makes.  All images live in one device byte arena
 * `base` (uint8 HWC BGR, packed); every offset below is a byte offset into it.  yolov6_b200/augment.py builds the tables.
 *
 * yv6_aug_resize: jobs [J][YV6_AUG_JOB] int64 = (src_off, h0, w0, dst_off, nh, nw, 0, 0): cv2.resize(INTER_LINEAR) of
 *   each source to nh x nw (a plain copy when the sizes are equal).  One launch serves load_image's resize of every source
 *   of a batch; a second launch over its results serves the letterbox branch's resize.  max_pix >= every nh * nw.
 * yv6_aug_resize_frames: the same resize (same jobs, same bytes) with job j's source read through srcs[j] (device [J]
 *   yv6_lb_src, layouts and pitches as for yv6_letterbox_frames) instead of base + src_off, which is ignored: a frame
 *   anywhere in device memory -- a decoder's output, a crop view, a frame cache.  The output is always packed BGR HWC at
 *   base + dst_off, so a job with (nh, nw) == (h0, w0) copies the frame into the arena in the layout yv6_augment reads.
 * yv6_augment: samples [B] (yv6_aug_sample, device) -> dst uint8 NCHW RGB [B,3,H,W].  Per output pixel: the flips as an
 *   index remap, then for each canvas cv2.warpAffine's INTER_LINEAR / BORDER_CONSTANT 114 sample of a virtual canvas --
 *   a 114 background of ch x cw with ntile placed rectangles, later tiles over earlier ones -- the fp64 mixup blend, and
 *   augment_hsv's BGR -> HSV -> LUT -> BGR.  W % 32 == 0 (OpenCV's vector HSV path then covers whole rows), dst
 *   16-byte aligned.
 * ---------------------------------------------------------------------------------------------- */
#define YV6_AUG_JOB 8
typedef struct {
  int64_t org;                 /* arena offset of canvas pixel (0, 0) in this tile's image (may lie outside the image) */
  int32_t pitch;               /* image width in pixels */
  int32_t y0, y1, x0, x1;      /* the tile's canvas rectangle [y0, y1) x [x0, x1) */
  int32_t pad;
} yv6_aug_tile;
typedef struct {
  double minv[2][6];           /* per canvas: M[:2] inverted as cv::warpAffine inverts it (dst -> canvas) */
  double mix_r;                /* mixup: trunc(c0 * r + c1 * (1 - r)) in fp64 */
  yv6_aug_tile tile[2][4];
  int32_t ch[2], cw[2];        /* canvas sizes */
  int32_t ntile[2];
  int32_t mixup, hsv, flipud, fliplr;
  uint8_t lut[3][256];         /* augment_hsv's hue, saturation and value tables */
} yv6_aug_sample;
int yv6_aug_resize(yv6_handle* h, uint8_t* base, const int64_t* jobs, int32_t J, int64_t max_pix, void* stream);
int yv6_aug_resize_frames(yv6_handle* h, const yv6_lb_src* srcs, const int64_t* jobs, int32_t J, int64_t max_pix,
                          uint8_t* base, void* stream);
int yv6_augment(yv6_handle* h, const uint8_t* base, const yv6_aug_sample* samples, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training-side irregular work: target preprocessing, label assignment, fused loss.
 * Compact assignment format shared by the assigners and the loss:
 *   gt      [B,G,5] float64  (class, x1, y1, x2, y2 in pixels; pad rows = -1,0,0,0,0)
 *   gt_idx  [B,A]   int32    assigned gt row (0 for background, as in the reference)
 *   fg      [B,A]   uint8    foreground mask
 *   norm    [B,A]   float64  target score of the assigned class (TAL: normalised alignment metric,
 *                            ATSS: IoU(gt, pred)); 0 for background
 * ---------------------------------------------------------------------------------------------- */

/* ComputeLoss.preprocess (reference yolov6/models/losses/loss.py:184-192) on the device: ragged
 * targets [n,6] fp32 (img, cls, cx, cy, w, h normalised) -> gt [B,G,5] float64 and gt_count [B]
 * (rows per image; rows beyond G are dropped and show up as gt_count > G). */
int yv6_targets_pad(yv6_handle* h, const float* targets, int32_t n, int32_t B, int32_t G, float scale_w,
                    float scale_h, double* gt, int32_t* gt_count, void* stream);

int64_t yv6_assign_workspace_bytes(int32_t B, int32_t A, int32_t G);

/* TaskAlignedAssigner.forward (reference yolov6/assigners/tal_assigner.py:22-173,
 * assigner_utils.py:25-89).  pd_scores [B,A,nc] fp32, pd_bboxes [B,A,4] fp32 xyxy pixels,
 * anc_points [A,2] fp32 pixels, mask_gt [B,G] uint8. */
int yv6_tal_assign(yv6_handle* h, const float* pd_scores, const float* pd_bboxes, const float* anc_points,
                   const double* gt, const uint8_t* mask_gt, int32_t B, int32_t A, int32_t G, int32_t nc,
                   int32_t topk, double alpha, double beta, double eps, int32_t* gt_idx, uint8_t* fg,
                   double* norm, void* workspace, int64_t workspace_bytes, void* stream);

/* ATSSAssigner.forward (reference yolov6/assigners/atss_assigner.py:18-161): anc_bboxes [A,4] fp32,
 * n_level_bboxes = HOST array of per-level anchor counts, pd_bboxes [B,A,4] fp32 pixels or NULL. */
int yv6_atss_assign(yv6_handle* h, const float* anc_bboxes, const int32_t* n_level_bboxes, int32_t nl,
                    const double* gt, const uint8_t* mask_gt, const float* pd_bboxes, int32_t B, int32_t A,
                    int32_t G, int32_t nc, int32_t topk, int32_t* gt_idx, uint8_t* fg, double* norm,
                    void* workspace, int64_t workspace_bytes, void* stream);

/* Dense (reference-shaped) assigner outputs for the drop-in API: labels int64 [B,A], bboxes float64
 * [B,A,4], scores float64 [B,A,nc], fg uint8 [B,A].  bg_label < 0: TAL convention (background keeps
 * gt 0's clamped label, tal_assigner.py:159-165); bg_label >= 0: ATSS (background = bg_label). */
int yv6_assign_expand(yv6_handle* h, const double* gt, const int32_t* gt_idx, const uint8_t* fg,
                      const double* norm, int32_t B, int32_t A, int32_t G, int32_t nc, int32_t bg_label,
                      int64_t* labels, double* bboxes, double* scores, uint8_t* fg_out, void* stream);

/* ComputeLoss.bbox_decode (loss.py:194-198) + dist2bbox (utils/general.py:32-38): pred_distri
 * [B,A,reg_ch] -> boxes [B,A,4] xyxy in stride units, or pixels when scale_to_pixels != 0
 * (the `pred_bboxes * stride_tensor` handed to the assigners, loss.py:94,100). strides: [A] fp32. */
int yv6_box_decode(yv6_handle* h, const float* pred_distri, const float* anc_points, const float* strides,
                   int32_t B, int32_t A, int32_t reg_ch, int32_t scale_to_pixels, float* boxes, void* stream);

/* Fused VFL + IoU (giou/siou/ciou/diou) + DFL loss, forward and backward (loss.py:157-182, 201-278;
 * utils/figure_iou.py:23-100).  out (device float64[8]): [0] loss, [1] w_iou*iou, [2] w_dfl*dfl,
 * [3] w_cls*cls (= reference loss_items order), [4] target_scores_sum, [5] num_pos.
 * grad_* receive d(loss * grad_scale)/d(pred_*), fp32, every element written. */
typedef struct yv6_loss_desc {
  const float* pred_scores;  /* [B,A,nc] post-sigmoid */
  const float* pred_distri;  /* [B,A,reg_ch] */
  const float* anc_points;   /* [A,2] pixels */
  const float* strides;      /* [A] */
  const double* gt;          /* [B,G,5] */
  const int32_t* gt_idx;
  const uint8_t* fg;
  const double* norm;
  int32_t B, A, G, nc, reg_ch;
  int32_t iou_type;          /* 0 giou, 1 siou, 2 ciou, 3 diou */
  double w_cls, w_iou, w_dfl;
  double grad_scale;
  float* grad_scores;
  float* grad_distri;
  double* out;
  void* workspace;
  int64_t workspace_bytes;   /* >= yv6_det_loss_workspace_bytes(B, A) */
  int32_t norm_gt_zero;      /* ABI 3: 0 = divide the sums by target_scores_sum when it is > 1 (loss.py:168-169, 238-262);
                              * 1 = when it is > 0, the rule of the fuse_ab loss (loss_fuseab.py:139, 203-206) */
} yv6_loss_desc;
int64_t yv6_det_loss_workspace_bytes(int32_t B, int32_t A);
int yv6_det_loss(yv6_handle* h, const yv6_loss_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * fuse_ab: the anchor-aided training branch of the head (effidehead_fuseab.py:94-140, loss_fuseab.py:58-76; SURVEY 8f N3).
 * Per level the two extra pred convs (yv6_conv_fwd, fp32 outputs, sigmoid fused on the class branch) write the natural
 * order raw_cls [B, hw, na*nc] / raw_reg [B, hw, na*4]; na = 3.
 * yv6_head_ab_pack:  -> rows [row_off + a*hw + p] of cls_ab [B, rows_total, nc] and reg_ab [B, rows_total, 4] =
 *                    (x_off, y_off, (2 sigmoid(r_w))^2 * anchors_wh[2a], (2 sigmoid(r_h))^2 * anchors_wh[2a+1]); anchors_wh = host
 *                    float[6], anchors_init of the level / stride (effidehead_fuseab.py:35,117-119).  row_off = 3 * (A of lower levels).
 * yv6_head_ab_grad:  gradients w.r.t. those tensors -> dense NHWC bf16 gradients w.r.t. the raw conv outputs
 *                    dl_cls [B, hw, cls_pad], dl_reg [B, hw, reg_pad] (sigmoid backward included, padded channels zero).
 * yv6_ab_boxes:      reg_ab + cell centres (pixels) + strides -> boxes in pixels (xyxy, for the assigner) and the equivalent
 *                    (l, t, r, b) distances in stride units, which yv6_det_loss consumes like an anchor-free head's output.
 * yv6_ab_boxes_bwd:  gradient w.r.t. (l, t, r, b) -> gradient w.r.t. (x_off, y_off, w, h).
 * ---------------------------------------------------------------------------------------------- */
int yv6_head_ab_pack(yv6_handle* h, const float* raw_cls, const float* raw_reg, int32_t B, int32_t hw, int32_t na, int32_t nc,
                     const float* anchors_wh, int32_t row_off, int32_t rows_total, float* cls_ab, float* reg_ab, void* stream);
int yv6_head_ab_grad(yv6_handle* h, const float* grad_cls_ab, const float* cls_ab, const float* grad_reg_ab, const float* raw_reg,
                     int32_t B, int32_t hw, int32_t na, int32_t nc, const float* anchors_wh, int32_t row_off, int32_t rows_total,
                     int32_t cls_pad, int32_t reg_pad, void* dl_cls, void* dl_reg, void* stream);
int yv6_ab_boxes(yv6_handle* h, const float* reg_ab, const float* anc_points, const float* strides, int32_t B, int32_t A,
                 float* ltrb, float* boxes_px, void* stream);
int yv6_ab_boxes_bwd(yv6_handle* h, const float* grad_ltrb, int64_t rows, float* grad_reg_ab, void* stream);

/* Self-distillation terms (losses/loss_distill.py:213-222 distill_loss_cls, :351-361 distill_loss_dfl): over `rows` rows of C
 * fp32 "logits" (student / teacher, contiguous), adds  eff * sum_rows KL(softmax(teacher/T) || softmax(student/T))  to *acc
 * (device double) and  eff * (softmax(student/T) - softmax(teacher/T)) / T  to grad (fp32, same shape as student; may be NULL).
 * row_mask (may be NULL): row r takes part iff row_mask[r / rows_per_mask] != 0 (the 4 sides of positive anchors).
 * eff = scale; if count_ptr != NULL: scale / (rows_per_mask * *count_ptr) (mean over the active rows, count on the device);
 * if gate_ptr != NULL and *gate_ptr <= 0: 0. */
int yv6_kl_rows(yv6_handle* h, const float* student, const float* teacher, int64_t rows, int32_t C, float temperature,
                const uint8_t* row_mask, int32_t rows_per_mask, double scale, const double* count_ptr, const double* gate_ptr,
                double* acc, float* grad, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training of the conv stack (train form): what autograd + cuDNN do for the reference's
 * Trainer.train_in_steps (yolov6/core/engine.py:142-176) under ConvModule.forward (conv -> BN(batch
 * stats) -> act, layers/common.py:46-49) and RepVGGBlock.forward (three BN-ed branches, common.py:245-255).
 * Forward = yv6_conv_fwd (no bias / act) + yv6_bn_stats + yv6_bn_finalize + yv6_bn_apply_fwd;
 * backward = yv6_bn_bwd -> yv6_conv_fwd with transposed / rotated weights (dgrad) + yv6_conv_wgrad.
 * ---------------------------------------------------------------------------------------------- */

/* dW[co][r][s][ci] (fp32 KRSC, ACCUMULATED into -- zero it first) from x [N,H,W,Cin] and dy [N,Ho,Wo,Cout]. */
typedef struct yv6_wgrad_desc {
  const void* x;  int32_t N, H, W, Cin, x_c_total;      /* bf16 NHWC (channel slice of a wider buffer allowed) */
  const void* dy; int32_t Cout, dy_c_total;             /* bf16 NHWC gradient of the conv output               */
  int32_t kh, kw, stride, pad;
  float* dw;                                            /* fp32 [Cout][kh][kw][Cin]                            */
  int32_t force_ksplit;                                 /* 0 = auto                                            */
  int32_t force_taps;                                   /* ABI 2: 0 = auto (3x3: one CTA accumulates a filter row), 1 = one tap per CTA */
} yv6_wgrad_desc;
int yv6_conv_wgrad(yv6_handle* h, const yv6_wgrad_desc* d, void* stream);
/* Host-only: the plan yv6_conv_wgrad makes for a device with the stated properties, no CUDA call.  out[0..9] = NT (Cin tile),
 * T (taps per CTA), PT (pixels per stage), BW, BH (pixel box), pixel tiles, ksplit (CTAs that add partial sums of the same dW
 * elements with fp32 atomics), pixels per split (PT * pixel tiles of the largest split, zero-filled rows included), CTAs,
 * dynamic shared memory in bytes. */
int yv6_wgrad_plan_host(int num_sms, int max_smem_optin, const yv6_wgrad_desc* d, int32_t* out10);

/* Per-channel sum and sum of squares (float64) of an NHWC bf16 tensor slice with channel pitch `pitch`. */
int yv6_bn_stats(yv6_handle* h, const void* x, int64_t pixels, int32_t C, int64_t pitch, double* sum, double* sumsq,
                 void* stream);
/* mean / invstd (biased var + eps), scale = gamma*invstd, shift = beta - mean*scale, and the running-stat
 * update of nn.BatchNorm2d (momentum, unbiased var); running_* may be NULL. */
int yv6_bn_finalize(yv6_handle* h, const double* sum, const double* sumsq, double count, const float* gamma,
                    const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                    float* mean_out, float* invstd_out, float* scale, float* shift, int32_t C, void* stream);

/* Up to three BN-ed branches summed and activated (RepVGG: conv3x3, conv1x1, identity; ConvModule: one). */
typedef struct yv6_bn_desc {
  int32_t nb, act, C;
  int64_t pixels;
  const void* x[3];  int64_t x_pitch[3];                /* branch inputs (bf16 NHWC slices)                    */
  const float* mean[3]; const float* invstd[3]; const float* scale[3]; const float* shift[3];
  void* y; int64_t y_pitch;                             /* block output (fwd: written; bwd: unused)            */
  /* backward only */
  const void* dy; int64_t dy_pitch;                     /* gradient w.r.t. the block output                    */
  double* s1; double* s2[3];                            /* [C] out: sum dz (= dbeta of every branch), sum dz*xhat_b (= dgamma_b) */
  void* dx[3]; int64_t dx_pitch[3]; int32_t accumulate[3];  /* gradient w.r.t. each branch input              */
  /* optional BottleRep shortcut (common.py:600-617): y = act(z) + res_alpha * res; backward adds
   * res_alpha * dy into dres and writes sum(dy * res) to dalpha[0] */
  const void* res; int64_t res_pitch; float res_alpha;
  void* dres; int64_t dres_pitch; double* dalpha;
  /* ABI 2 */
  const float* res_alpha_dev;                           /* when set, the shortcut weight is read from this device scalar (no
                                                           host synchronisation, graph-capturable) instead of res_alpha      */
  /* scratch of the two-pass backward (optional; the handle's scratch is used when work == NULL): work [nb][C] float64,
   * counter one uint32, coef [nb][2][C] fp32.  zeroed != 0: the caller already zeroed s1, work, counter and dalpha
   * (the training engine clears one arena per step instead of four memsets per block). */
  double* work; uint32_t* counter; float* coef; int32_t zeroed;
  int32_t dres_assign;                                  /* != 0: dres = alpha * dy (first writer of that gradient slice) instead of += */
} yv6_bn_desc;
int yv6_bn_apply_fwd(yv6_handle* h, const yv6_bn_desc* d, void* stream);

/* Batch statistics of up to three branch inputs and their finalisation in ONE launch: per-channel sum / sum of squares
 * (float64 atomics of block-level partial sums), then -- in the thread block that finishes last -- mean, invstd,
 * scale = gamma*invstd, shift = beta - mean*scale and the running-statistics update of nn.BatchNorm2d for every branch
 * (ConvModule / RepVGGBlock in train mode, layers/common.py:46-49,245-255; eps / momentum of torch_utils.py:38-48). */
typedef struct yv6_bn_stats_desc {
  int32_t nb, C;
  int64_t pixels;
  const void* x[3]; int64_t x_pitch[3];                 /* bf16 NHWC slices                                              */
  double* sums;                                         /* [nb][2][C] sum, sumsq                                          */
  uint32_t* counter;                                    /* one uint32                                                     */
  int32_t zeroed;                                       /* != 0: sums and counter are already zero                        */
  const float* gamma[3]; const float* beta[3];
  float* running_mean[3]; float* running_var[3];        /* may be NULL                                                    */
  float* stats[3];                                      /* out [4][C]: mean, invstd, scale, shift; NULL = sums only       */
  float eps, momentum;
} yv6_bn_stats_desc;
int yv6_bn_stats_finalize(yv6_handle* h, const yv6_bn_stats_desc* d, void* stream);
int yv6_bn_bwd(yv6_handle* h, const yv6_bn_desc* d, void* stream);

/* QARepVGGBlock / QARepVGGBlockV2 (layers/common.py:322-477): the branch sum in front of the block's post-sum BatchNorm,
 *   t = scale_d * u + shift_d + v [+ x [+ avg3x3(x)]]
 * with u the raw 3x3 conv (BN_d = rbr_dense.bn), v the bare 1x1 conv, x the block input (identity, Cin == C at stride 1) and
 * avg3x3 = AvgPool2d(3, 1, 1), which divides by 9 at the border too.  Any C and channel pitch; channels outside [0, C) are
 * not written.
 * yv6_qa_fwd: writes t (bf16) and, in the same launch, the float64 per-channel sum / sum of squares of the ROUNDED t into
 *   sums [2][C] (zero on entry when zeroed != 0); the thread block that finishes last writes stats [4][C] = mean, invstd,
 *   scale = gamma * invstd, shift = beta - mean * scale of the post-sum bn and updates its running statistics (may be NULL),
 *   as yv6_bn_stats_finalize does.
 * yv6_qa_bwd: the identity / avg part of the input gradient, dx (+)= dt + avg3x3^T(dt) (accumulate != 0: +=). */
typedef struct yv6_qa_desc {
  int32_t N, H, W, C;
  const void* u; int64_t u_pitch;
  const void* v; int64_t v_pitch;
  const float* scale_d; const float* shift_d;           /* [C] each                                                        */
  const void* x; int64_t x_pitch;                       /* NULL: no identity / avg branch                                  */
  int32_t avg, accumulate;
  void* t; int64_t t_pitch;
  double* sums; uint32_t* counter; int32_t zeroed; float eps;
  const float* gamma; const float* beta;
  float* running_mean; float* running_var; float* stats; float momentum; int32_t reserved0;
  const void* dt; int64_t dt_pitch;                     /* backward: gradient w.r.t. t                                     */
  void* dx; int64_t dx_pitch;                           /* backward: gradient w.r.t. the block input                       */
} yv6_qa_desc;
int yv6_qa_fwd(yv6_handle* h, const yv6_qa_desc* d, void* stream);
int yv6_qa_bwd(yv6_handle* h, const yv6_qa_desc* d, void* stream);

/* Head gradients: level slice [off, off+hw) of the [B,A,ch] fp32 tensors -> dense NHWC bf16 [B,hw,ch_pad];
 * with `scores` the sigmoid backward dlogit = dscore * s * (1 - s) of effidehead.py:85 is applied. */
int yv6_head_grad_prep(yv6_handle* h, const float* grad, const float* scores_or_null, int32_t B, int32_t A, int32_t ch,
                       int32_t level_off, int32_t level_hw, int32_t ch_pad, void* out_bf16, void* stream);
/* Backward of one MaxPool2d(5,1,2) of SPPF (common.py:104-112): dx (+)= scatter of dy to the window arg-max. */
int yv6_maxpool5_bwd(yv6_handle* h, const void* x, int64_t x_pitch, const void* dy, int64_t dy_pitch, int32_t N,
                     int32_t H, int32_t W, int32_t C, float* dx_scratch, void* dx, int64_t dx_pitch, int32_t accumulate,
                     void* stream);
/* Weight gradient of the 3-channel stem conv (3x3 stride 2): dw fp32 [Cout][3][3][3] (overwritten). */
int yv6_stem_wgrad(yv6_handle* h, const void* x, int32_t x_dtype, float in_scale, const void* dy, int64_t dy_pitch,
                   int32_t N, int32_t H, int32_t W, int32_t Cout, float* dw, void* stream);

/* Both stem branches of a RepVGG stem in one pass over the image: dw3 fp32 [Cout][3][3][3] from dy3 and (optional) dw1 fp32
 * [Cout][3] (the 1x1 stride-2 branch = centre tap) from dy1; ACCUMULATED into (zeroed != 0: the caller cleared them). */
int yv6_stem_wgrad2(yv6_handle* h, const void* x, int32_t x_dtype, float in_scale, const void* dy3, int64_t dy3_pitch,
                    const void* dy1, int64_t dy1_pitch, int32_t N, int32_t H, int32_t W, int32_t Cout, float* dw3, float* dw1,
                    int32_t zeroed, void* stream);

/* im2col of the 3-channel stem conv (3x3, stride 2, pad 1): patches bf16 [N, Ho, Wo, 32] with channel (r*3+s)*3 + c =
 * x[n, c, 2ho+r-1, 2wo+s-1] (x as in yv6_stem_fwd: NCHW fp32 or uint8 * in_scale), channels 27..31 zero.  With it the stem's
 * weight gradient is a 1x1 yv6_conv_wgrad over (patches, dY): dw [Cout][32] fp32.  patches_lo (optional) receives the bf16
 * rounding residual of the patches; a second wgrad over it restores the fp32 image in the gradient. */
int yv6_stem_im2col(yv6_handle* h, const void* x, int32_t x_dtype, float in_scale, int32_t N, int32_t H, int32_t W,
                    void* patches_bf16, void* patches_lo_bf16, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Step-level plumbing of the training engine (SURVEY.md 8f N1/N2): everything that the reference does with
 * hundreds of small eager ops per step -- autocast weight casts, layout permutes, `.grad` accumulation,
 * torch.optim.SGD (solver/build.py:10-33) and ModelEMA.update (utils/ema.py:28-37) -- as three launches.
 * ---------------------------------------------------------------------------------------------- */
#define YV6_XFORM_CHUNK 4096
enum { YV6_XF_F32 = 0, YV6_XF_F64 = 1, YV6_XF_BF16 = 2 };
/* dst[d0*ds0 + d1*ds1 + d2*ds2 + d3*ds3] (+)= cast(src[d0*ss0 + d1*ss1 + d2*ss2 + d3*ss3]) for d in n[0] x n[1] x n[2] x n[3];
 * strides in elements, source strides may be negative (filter rotation for dgrad).  src: fp32 or float64; dst: bf16 or fp32. */
typedef struct yv6_xform_seg {
  void* dst; const void* src;
  int32_t n[4], ds[4], ss[4];
  int32_t dst_dtype, src_dtype;
} yv6_xform_seg;
/* segs / chunk tables live in DEVICE memory: chunk c of the launch works on segment chunk_seg[c], elements
 * [(c - chunk_first[seg]) * YV6_XFORM_CHUNK, +YV6_XFORM_CHUNK).  accumulate applies to fp32 destinations. */
int yv6_xform(yv6_handle* h, const yv6_xform_seg* segs_dev, const int32_t* chunk_seg_dev, const int32_t* chunk_first_dev,
              int32_t n_chunks, int32_t accumulate, void* stream);

/* SGD(momentum, nesterov) + weight decay + EMA over flat fp32 buffers of n elements (n % 4 == 0).  group_per4[i] is the
 * parameter group of elements 4i..4i+3: 0 = BN weights, 1 = conv weights (weight decay), 2 = biases, 3 = float buffers
 * (EMA only), 255 = padding.  hyper (device, 8 floats): lr[0..2], momentum, weight_decay, ema_decay, first_step, grad_scale.
 * ema_or_null == NULL skips the EMA update. */
int yv6_sgd_ema_step(yv6_handle* h, float* param, const float* grad, float* momentum_buf, float* ema_or_null,
                     const uint8_t* group_per4, int64_t n, const float* hyper_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Inference weight fold (yolov6_b200/refold.py): the train-form state in one flat fp32 buffer (flat.FlatState layout, or
 * a state_dict staged that way) -> every weight tensor of an inference engine, in place, bit for bit what fold.py's float64
 * fold and the engine's casts give on the host.  Two phases over records built on the host once per (engine, layout):
 *   channel phase: one yv6_fold_chan per op: the BatchNorm affine(s) of its branches in float64 -> coef[5 per channel] =
 *                  (A: main weight scale, B: 1x1 branch scale, D: identity term, P: post-sum scale, folded bias);
 *   element phase: one yv6_fold_rec per destination region: value(o, r, s, c) in float64, then cast to the region's format.
 * Every float64 operation is an explicit round-to-nearest intrinsic in fold.py's order (no FMA contraction).
 * ---------------------------------------------------------------------------------------------- */
#define YV6_FOLD_CHUNK 4096
enum { YV6_FOLD_C_DP = 0, YV6_FOLD_C_REP = 1, YV6_FOLD_C_QA = 2, YV6_FOLD_C_BN = 3, YV6_FOLD_C_BIAS = 4 };
/* element layouts: W: w * A; W_REP: w3 * A + (center ? w1 * B : 0) (+ D on the identity diagonal's center); W_QA:
 * ((w3 * A + (center ? w1 : 0)) (+ 1 on the diagonal's center) (+ 1/9 on the diagonal if avg)) * P; W_COPY: w; W_CONVT:
 * w[c][o][r0][s0] of a [Cin][Cout][2][2] ConvTranspose weight; BIAS: the folded bias of channel o; COPY: flat element o. */
enum { YV6_FOLD_W = 0, YV6_FOLD_W_REP = 1, YV6_FOLD_W_QA = 2, YV6_FOLD_W_COPY = 3, YV6_FOLD_W_CONVT = 4, YV6_FOLD_BIAS = 5,
       YV6_FOLD_COPY = 6 };
/* formats: fp32 (float64 -> fp32), bf16 (-> fp32 -> bf16), fp16 (-> fp32 -> fp16, as torch casts float64), split3 (-> fp32 ->
 * three bf16 planes hi / mid / lo, `plane_stride` elements apart, residuals in fp32) */
enum { YV6_FOLD_F32 = 0, YV6_FOLD_BF16 = 1, YV6_FOLD_F16 = 2, YV6_FOLD_SPLIT3 = 3 };
enum { YV6_FOLD_IDENTITY = 1, YV6_FOLD_AVG = 2 };
typedef struct yv6_fold_chan {
  int64_t bn[3][4];            /* flat offsets of (weight, bias, running_mean, running_var) of the op's BatchNorms at its first
                                  channel, -1: absent.  C_DP / C_BN: [0]; C_REP: dense, 1x1, identity; C_QA: dense, post-sum */
  int64_t b;                   /* flat offset of the conv bias (C_DP, C_BIAS), -1: absent */
  int64_t coef;                /* first coefficient of channel 0 (5 doubles per channel) */
  int32_t layout, n;           /* YV6_FOLD_C_*, channels */
} yv6_fold_chan;
typedef struct yv6_fold_rec {
  void* dst;                   /* destination element of domain point 0 */
  int64_t plane_stride;        /* split3: elements between the planes */
  int64_t ds[4];               /* destination strides (elements) of the domain axes (o, r, s, c) */
  int64_t w, w1;               /* flat offsets of the op's weight at its first output channel and of the rep / qa 1x1 weight, -1: absent */
  int64_t coef;                /* first coefficient of channel 0 */
  int64_t blk0;                /* first block of the element phase working on this record (records in increasing blk0) */
  int32_t n[4];                /* domain: output channels, tap rows, tap columns, input channels */
  int32_t layout, fmt;         /* YV6_FOLD_W*, YV6_FOLD_F* */
  int32_t k, cin;              /* the weight's kernel size and input channels (per group) */
  int32_t r0, s0;              /* tap of domain point (r, s) = 0 (column-pair view columns, ConvTranspose quadrant) */
  int32_t cout;                /* W_CONVT: the weight's output channels */
  int32_t flags;               /* YV6_FOLD_IDENTITY | YV6_FOLD_AVG */
  int32_t check;               /* fp16 range check slot, -1: none */
  int32_t reserved0;
} yv6_fold_rec;
/* Records and coef live in DEVICE memory; n_blocks = blk0 of a record past the last.  check_only == 0: both phases, every
 * record written.  check_only == 1: the channel phase, then the element values of the records with a check slot are rounded
 * to fp16 (through fp32) and nothing but coef and `checks` is written: checks[2 * slot] |= 1 if one is not finite,
 * checks[2 * slot + 1] = max of the bits of |value| (the float64 max |value|); the caller zeroes `checks` first. */
int yv6_fold(yv6_handle* h, const float* flat, const yv6_fold_chan* chans_dev, int32_t n_chans, const yv6_fold_rec* recs_dev,
             int32_t n_recs, int64_t n_blocks, double* coef, unsigned long long* checks, int32_t check_only, void* stream);

/* ---- JPEG decode (yv6_jpeg.cu): cv2.imread's pixels of baseline / extended sequential Huffman JPEGs ----
 * The host parses each header (yolov6_b200/jpeg.py) into one yv6_jpeg_image; one call decodes a batch of them.
 * yv6_jpeg_huff: one Huffman table: lut[x] = length << 8 | symbol for the codes of at most 9 bits (x: the next 9 bits),
 *   0 otherwise; maxcode[l] the largest l-bit code (-1: none, [17] a sentinel), vals[code + valoff[l]] its symbol.
 * yv6_jpeg_comp / yv6_jpeg_image: the caller fills the fields marked (in); yv6_jpeg_workspace_bytes fills the rest. */
typedef struct yv6_jpeg_huff {
  uint16_t lut[512];
  int32_t maxcode[18];
  int32_t valoff[18];
  uint8_t vals[256];
} yv6_jpeg_huff;
typedef struct yv6_jpeg_comp {
  int32_t h, v;                /* (in) sampling factors                                                          */
  int32_t dc, ac;              /* (in) indices of its tables in the call's yv6_jpeg_huff array                    */
  int32_t bw, bh;              /* plane size in blocks                                                            */
  int32_t dw, dh;              /* real samples of the plane: ceil(width * h / hmax), ceil(height * v / vmax)       */
  int64_t plane;               /* workspace offset of the (bw * 8) x (bh * 8) uint8 sample plane                  */
  uint16_t q[64];              /* (in) quantisation table, natural order                                         */
} yv6_jpeg_comp;
typedef struct yv6_jpeg_image {
  const uint8_t* data;         /* (in) the entropy-coded segment, device memory (after SOS, up to the next non-RST marker) */
  int64_t len;                 /* (in) its bytes                                                                  */
  uint8_t* out;                /* (in) height x width x 3 BGR uint8 (width x height x 3 for orientations 5-8)      */
  int32_t height, width;       /* (in) the frame as coded                                                         */
  int32_t ncomp;               /* (in) 1 or 3                                                                    */
  int32_t orientation;         /* (in) EXIF orientation 1..8, applied as cv2.imread does                          */
  int32_t restart;             /* (in) MCUs per restart interval, 0: none (set to every MCU)                      */
  int32_t mcux, mcuy, nblk;    /* MCUs per row and column, blocks per MCU                                         */
  int64_t ws_bytes;            /* workspace offsets: the unstuffed segment (len + 16 bytes),                      */
  int64_t ws_rst;              /*   the start bit of each restart interval and the end (int64),                   */
  int64_t ws_coef;             /*   the coefficients, 64 int16 per block in scan order                            */
  yv6_jpeg_comp comp[3];
} yv6_jpeg_image;
enum { YV6_JPEG_OK = 0, YV6_JPEG_SHORT = 1, YV6_JPEG_BAD_CODE = 2, YV6_JPEG_BAD_RUN = 3 };
/* Host function: lays out the per-call workspace of imgs[0..n) (host records), filling their derived fields; returns its
 * bytes, or -1 with yv6_last_error set when a record is not one the decoder takes. */
int64_t yv6_jpeg_workspace_bytes(yv6_jpeg_image* imgs, int32_t n);
/* Decodes imgs[0..n) (records and tables in DEVICE memory, laid out by yv6_jpeg_workspace_bytes) into their `out` frames.
 * status[i] (device int32) becomes YV6_JPEG_OK or the first error found in image i's entropy data (its pixels are then
 * unspecified); nothing is read outside the segments, the tables and the workspace.  The host is never synchronised. */
int yv6_jpeg_decode(yv6_handle* h, const yv6_jpeg_image* imgs, int32_t n, const yv6_jpeg_huff* huff, void* workspace,
                    int32_t* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YV6_H_ */
