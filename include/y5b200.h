/* y5b200.h -- C ABI of liby5b200.so: the H100 (sm_90a) engine behind the YOLOv5 forward / NMS / loss hot path.
 *
 * The reference (ultralytics/yolov5) is pure Python and has NO FFI / plugin interface for this path: the work
 * sits behind ordinary Python callables (SURVEY.md section 8b).  Each entry point below therefore names the
 * reference callable whose body it replaces (file:line under /root/reference); INTEGRATION.md shows the ctypes
 * stubs a maintainer adds to those files.
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes only; device pointers are raw CUDA device addresses; `stream` is a cudaStream_t;
 *   - never allocate device memory, never synchronise the stream, never touch the default stream;
 *   - activations are NHWC ("pixel-major"): element (n,y,x,c) of a view lives at base[((n*H+y)*W+x)*pitch + c],
 *     where `pitch` (elements per pixel of the underlying buffer) >= the view's channel count -- a view may be a
 *     channel slice of a wider buffer (this is how torch.cat is eliminated); pitches and channel offsets are
 *     multiples of 8 elements (16 bytes);
 *   - dtype: Y5_F16 or Y5_BF16 for activations and packed weights; accumulation and bias are fp32;
 *   - return 0 on success, a negative Y5_E* code for a rejected argument, a positive cudaError_t for a CUDA
 *     failure; y5_last_error() returns a thread-local message for the last non-zero return.
 */
#ifndef Y5B200_H
#define Y5B200_H
#include <stdint.h>

#if defined(__GNUC__)
#define Y5_API __attribute__((visibility("default")))
#else
#define Y5_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define Y5_F16 0
#define Y5_BF16 1
#define Y5_F32 2
#define Y5_U8 3

#define Y5_E_INVALID (-1)     /* bad argument (null pointer, misaligned pitch, ...) */
#define Y5_E_UNSUPPORTED (-2) /* shape outside what the kernels implement */
#define Y5_E_DRIVER (-3)      /* tensor-map encode / driver entry point unavailable */

#define Y5_ACT_NONE 0
#define Y5_ACT_SILU 1
#define Y5_ACT_LEAKY 2 /* v > 0 ? v : slope * v in fp32 (nn.LeakyReLU(slope); nn.ReLU is slope 0), slope passed next to the code */

int y5_version(void);
const char* y5_last_error(void);
/* number of kernel launches issued through this library since load (bench.py's gpu_launches) */
int64_t y5_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused Conv2d(bias=False) + folded BatchNorm + SiLU or LeakyReLU / ReLU (+ residual add), implicit GEMM on wgmma tensor cores.
 * The activation (desc.act, desc.act_slope) acts on fp32(acc + bias); the residual is added in fp32 and the sum rounded once.
 * Replaces: models/common.py:86-92 Conv.forward / forward_fuse (conv -> bn -> act), utils/torch_utils.py:224-254
 * (BN fold, done once by the caller when packing), models/common.py:181 Bottleneck's `x + ...` (residual),
 * and, through out pitch/offset, the torch.cat of models/common.py:246,340,453.
 *   weights : packed [out_c][kh][kw][cin_pad] (K-major), cin_pad = chunks*block_k as reported by y5_conv_pick,
 *             zero padded, dtype = activation dtype, BN scale already folded in
 *   bias    : fp32 [out_c] (folded BN shift)
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct y5_conv_desc {
    const void* in;       /* view base (already offset to its first channel) */
    int32_t in_pitch;     /* elements per pixel of the buffer holding the view */
    int32_t batch, in_h, in_w, in_c;
    const void* weight;
    const float* bias;
    void* out;            /* view base (already offset to its first channel) */
    int32_t out_pitch;
    int32_t out_c;
    const void* residual; /* optional: same shape as out; may alias out (in-place add) */
    int32_t res_pitch;
    int32_t ksize, stride, pad;
    int32_t act;          /* Y5_ACT_NONE | Y5_ACT_SILU | Y5_ACT_LEAKY (with act_slope) */
    int32_t dtype;        /* Y5_F16 | Y5_BF16 */
    int32_t block_k;      /* 16|32|64, or 0 = y5_conv_pick's choice; must match the weight packing */
    int32_t block_n;      /* 32|64|128|256, or 0 = auto */
    /* optional generalisations (all 0 = the plain case above) */
    int32_t kw;           /* non-square filter: width (height stays `ksize`); 0 = square, and then pad_w is ignored */
    int32_t pad_w;        /* horizontal padding, only read when kw != 0 (vertical padding stays `pad`) */
    int64_t in_x_stride;  /* elements between horizontally adjacent pixels (0 = in_pitch).  A stride smaller than in_c
                             exposes overlapping "wide pixels": the stem runs as a 3x1 conv over 48-channel pixels
                             that each span 3 neighbouring 16-channel space-to-depth cells */
    int64_t in_y_stride;  /* elements between rows   (0 = in_w * in_x_stride) */
    int64_t in_n_stride;  /* elements between images (0 = in_h * in_y_stride) */
    int32_t a_mode;       /* activation fetch: 0 auto, 1 force TMA-im2col, 2 force shifted-patch (stride-1 only) */
    int32_t reserved;     /* flags, 0 in normal use.  Tuning / tests: bit 3 (8) staged epilogue (each warpgroup's block goes
                             through shared memory and leaves as 16-byte row segments), bit 4 (16) forces direct register
                             stores instead of the default TMA epilogue; bit 7 (128) the wide patch fetch (one patch copy per channel chunk
                             feeds every tap of a stride-1 k x k conv with 64-channel chunks), bit 5 (32) vetoes it; with a
                             forced block_n also bit 1 (2) = 256-row tiles (block_n 128), bit 2 (4) = CTA pairs (2-CTA cluster),
                             bits 8.. = cluster size (2|4): the CTAs of a cluster split every weight tile and TMA-multicast it */
    float act_slope;      /* Y5_ACT_LEAKY: negative slope (finite; 0 = ReLU).  Ignored for the other activations */
} y5_conv_desc;

/* Tiling the library will use for a conv: block_k decides the weight packing (cin_pad = ceil(in_c/block_k)*block_k). */
int y5_conv_pick(int32_t in_c, int32_t out_c, int64_t m_rows, int32_t* block_k, int32_t* block_n);

typedef struct y5_conv_plan y5_conv_plan; /* opaque: encoded TMA descriptors + launch geometry for fixed pointers */
int y5_conv_plan_create(const y5_conv_desc* desc, y5_conv_plan** plan);
int y5_conv_plan_run(const y5_conv_plan* plan, void* stream);
void y5_conv_plan_destroy(y5_conv_plan* plan);
/* What a plan will run (read-only; tests assert the kernel path a case claims through it).  A plain struct tag, not a
 * typedef: the query function has the same name. */
struct y5_conv_plan_info {
    int32_t a_mode;               /* activation fetch: 0 LINEAR (1x1/s1 GEMM), 1 TMA-im2col, 2 shifted patch */
    int32_t tw, th;               /* patch: output pixels per tile row x rows (tw * th = 128); 0 in the other modes */
    int32_t block_k, block_n, mt; /* K block, N tile, 128-row sub-tiles per tile */
    int32_t cluster;              /* CTAs per cluster sharing (multicasting) every weight tile: 1, 2 or 4 */
    int32_t patch_pw;             /* > 0: wide patch (one patch copy per channel chunk feeds every tap), its row pitch */
    int32_t b_grouped;            /* patch: the kh weight tiles of a (chunk, horizontal tap) group share one stage */
    int32_t staged;               /* epilogue stores go through shared memory (else straight from the registers) */
    int32_t opt;                  /* runs the kernel instantiation with the optional modes compiled in */
    int32_t epi;                  /* epilogue: 0 conv (SiLU or none), 1 Detect head, 2 conv with LeakyReLU / ReLU */
    int32_t a_stages, b_stages;   /* shared-memory pipeline depth */
    int32_t grid;                 /* CTAs launched (persistent, at most one per SM) */
    int32_t tma_epi;              /* epilogue through shared memory: residual TMA-loaded, output TMA-stored */
};
int y5_conv_plan_info(const y5_conv_plan* plan, struct y5_conv_plan_info* info);
/* one-shot convenience: create + run + destroy (tests) */
int y5_conv_bn_silu_fwd(const y5_conv_desc* desc, void* stream);
/* independent direct-convolution kernel (CUDA cores, fp32 accumulate) used by tests to cross-check the tensor-core
 * path on the device; same descriptor, weights in the same packed layout */
int y5_conv_direct_fwd(const y5_conv_desc* desc, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Detect / Segment head level: 1x1 conv with bias + reshape + sigmoid/grid/anchor decode in the GEMM epilogue.
 * Replaces models/yolo.py:95-113 for one level i (conv, view/permute, sigmoid, xy/wh decode, cat into z).
 *   raw : (B, na, ny, nx, no)  un-activated logits, activation dtype            (x[i] of the reference)
 *   z   : (B, z_rows, no) decoded rows; this level writes rows [z_row0, z_row0 + na*ny*nx) of every image
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct y5_detect_desc {
    const void* in;
    int32_t in_pitch;
    int32_t batch, ny, nx, in_c;
    const void* weight;   /* packed [na*npad][cin_pad], npad = 128 * ceil(no / 128): anchor a in rows [a*npad, a*npad + no),
                             the rest zero (npad = 128 while no <= 128) */
    const float* bias;    /* fp32 [na*npad], laid out like the weight rows */
    int32_t z_rows, z_row0;
    int32_t na, no, nc;   /* no = 5 + nc + nm <= 8192, nc <= 4096 (Y5_E_UNSUPPORTED beyond); columns >= 5+nc (mask
                             coefficients) are passed through un-sigmoided */
    float stride;         /* pixels per cell of this level */
    float anchor_wh[8];   /* na x (w,h) in PIXELS (= anchors * stride), na <= 4 */
    int32_t dtype;
    int32_t block_k;
} y5_detect_desc;
typedef struct y5_detect_plan y5_detect_plan;
int y5_detect_plan_create(const y5_detect_desc* desc, y5_detect_plan** plan);
/* runs the plan into the outputs given per call (the reference returns new tensors from every forward; the input side
 * of the plan stays bound to the engine's static buffers) */
int y5_detect_plan_run_to(const y5_detect_plan* plan, void* raw, void* z, void* stream);
void y5_detect_plan_destroy(y5_detect_plan* plan);

/* ---------------------------------------------------------------------------------------------------------------
 * Data-movement kernels (HBM bound)
 * ------------------------------------------------------------------------------------------------------------- */
/* Stem input: NCHW image (Y5_U8 scaled by 1/255, or Y5_F16/Y5_BF16/Y5_F32 already in [0,1]) -> 2x2 space-to-depth
 * NHWC with 16 channels (12 used: (dy*2+dx)*3 + c; 4 zero), so that the 6x6/s2/p2 stem conv of
 * models/yolov5s.yaml:20 becomes a 3x3/s1/p1 conv over 16 channels.  Replaces the `im.half(); im /= 255` of
 * detect.py:206-208 / val.py:259-262 plus the layout change.  h, w even.  `out_row_px` (0 = w/2) is the number of
 * 16-channel cells per output row of the buffer and `out_x_off` the cell where each row starts: the engine keeps one
 * zero cell left and right of every row so the stem conv can read 3 neighbouring cells as one 48-channel pixel.
 * `out` must be 16-byte aligned (Y5_E_INVALID otherwise). */
int y5_stem_s2d(const void* img, int32_t img_dtype, void* out, int32_t out_dtype, int32_t batch, int32_t h, int32_t w,
                int32_t out_row_px, int32_t out_x_off, void* stream);
/* Input of a first layer that is not the v6 stem (models/hub/yolov3*.yaml start with Conv(3, c, 3, 1)): NCHW image (dtypes
 * as y5_stem_s2d) -> dense NHWC [batch][h][w][out_c] in out_dtype (fp16/bf16), channels 0..2 the image and 3..out_c-1
 * zero.  out_c a multiple of 8; `out` 16-byte aligned. */
int y5_image_nhwc(const void* img, int32_t img_dtype, void* out, int32_t out_dtype, int32_t batch, int32_t h, int32_t w,
                  int32_t out_c, void* stream);
/* SPPF pooling (models/common.py:338-340): reads view x (c channels), writes maxpool5, maxpool5^2 (=9x9),
 * maxpool5^3 (=13x13) into three views (usually channel slices 1..3 of the buffer whose slice 0 is x).  A NaN in a
 * window makes its maximum NaN, as F.max_pool2d does.  y5_sppf_pool, y5_upsample2x and y5_copy_view move 16-byte
 * vectors: every view must be 16-byte aligned with pitch >= c (Y5_E_INVALID otherwise), c and pitches multiples of 8. */
int y5_sppf_pool(const void* x, int32_t x_pitch, void* y1, void* y2, void* y3, int32_t y_pitch, int32_t batch, int32_t h,
                 int32_t w, int32_t c, int32_t ksize, int32_t dtype, void* stream);
/* nn.Upsample(scale_factor=2, mode='nearest') written straight into a (concat) view. */
int y5_upsample2x(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                  int32_t dtype, void* stream);
/* strided channel-slice copy (only needed when a tensor feeds two concat buffers) */
int y5_copy_view(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int64_t pixels, int32_t c, int32_t dtype,
                 void* stream);
/* NHWC view -> dense NCHW tensor (the API hands NCHW tensors back to PyTorch callers, e.g. Segment's proto) */
int y5_nhwc_to_nchw(const void* x, int32_t x_pitch, void* y, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t dtype,
                    void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * non_max_suppression (utils/general.py:658-767) for a whole batch in one launch set; bit-exact indices.
 *   pred     : (B, N, no) decoded predictions, dtype Y5_F16 | Y5_BF16 | Y5_F32, dense
 *   classes  : optional device array of class ids to keep (int32), n_classes entries
 *   out_rows : (B, max_det, 6+nm) fp32   [x1,y1,x2,y2,conf,cls,masks...]
 *   out_idx  : (B, max_det) int64        candidate id = row*nc + cls of each kept detection
 *   out_count: (B) int32                 detections kept per image
 *   workspace: y5_nms_workspace_bytes(...) bytes of scratch
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct y5_nms_params {
    int32_t batch, n_rows, no, nc, nm;
    int32_t dtype;
    float conf_thres, iou_thres;
    int32_t multi_label, agnostic;
    int32_t max_det;  /* reference default 300 */
    int32_t max_nms;  /* reference constant 30000 */
    float max_wh;     /* reference constant 7680 */
    const int32_t* classes;
    int32_t n_classes;
} y5_nms_params;
int64_t y5_nms_workspace_bytes(const y5_nms_params* p);
int y5_nms_batched(const y5_nms_params* p, const void* pred, float* out_rows, int64_t* out_idx, int32_t* out_count,
                   void* workspace, int64_t workspace_bytes, void* stream);
/* box_iou (ultralytics.utils.metrics.box_iou as used by utils/metrics.py:158,252): (n,4) x (m,4) -> (n,m), fp32 */
int y5_box_iou(const float* a, int32_t n, const float* b, int32_t m, float eps, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * ComputeLoss (utils/loss.py:134-247): build_targets + gather/CIoU/scatter + BCE, forward and backward.
 *   p[l]      : (B, na, ny_l, nx_l, no) logits, dtype Y5_F16 | Y5_BF16 | Y5_F32
 *   targets   : (nt, 6) fp32 [img, cls, x, y, w, h]
 *   anchors   : (nl, na, 2) fp32, grid units
 *   out_loss  : fp32[4] = [loss*bs, lbox, lobj, lcls]  (gains already applied)
 *   grad[l]   : optional, same shape AND dtype as p[l]: d(out_loss[0] * grad_scale)/dp  (fully written)
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct y5_loss_params {
    int32_t nl, batch, na, no, nc;
    int32_t ny[5], nx[5];
    int32_t dtype;
    int32_t nt;
    float anchor_t, box_gain, obj_gain, cls_gain, cls_pw, obj_pw, cp, cn;
    float balance[5];
    float grad_scale;
} y5_loss_params;
int64_t y5_loss_workspace_bytes(const y5_loss_params* p);
/* matches: per level, int32 count + rows (b, a, gj, gi, cls) int64 and tbox fp32 live in the workspace; the
 * build_targets result can be read back with y5_loss_read_targets for parity tests.
 * The upstream gradient of the loss is read from DEVICE memory: grad[l] = d(out_loss[0])/dp * p->grad_scale *
 * (*grad_scale_dev), multiplied in fp32 BEFORE the result is rounded to the prediction dtype -- what autograd does for
 * `scaler.scale(loss).backward()` (train.py:410): a GradScaler factor of 65536 (x WORLD_SIZE) neither overflows fp16 on
 * the way nor flushes small objectness gradients to zero.  grad_scale_dev may be NULL (= 1).  Targets whose image index
 * is outside [0, batch) or whose class is outside [0, nc) are ignored (the reference raises IndexError for them). */
int y5_loss_fwd_bwd_scaled(const y5_loss_params* p, const void* const* pl, const float* targets, const float* anchors,
                           float* out_loss, void* const* grad, const float* grad_scale_dev, void* workspace,
                           int64_t workspace_bytes, void* stream);
int y5_loss_read_targets(const y5_loss_params* p, const void* workspace, int32_t level, int64_t* idx5_host,
                         float* tbox_host, int32_t* count_host, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Segmentation ComputeLoss (utils/segment/loss.py:48-195): the detection terms above plus the cropped mask BCE.
 *   p[l]       : (B, na, ny_l, nx_l, no) logits with no == 5 + nc + nm; p->batch <= 1024
 *   proto      : (B, nm, mh, mw) of proto_dtype, element strides ps_* of a dense layout (NCHW or channels_last, no
 *                gaps: grad_proto is written at the same offsets); nm <= 32
 *   masks      : (n_masks, gt_h, gt_w) fp32 contiguous; overlap: n_masks == batch and pixel value v marks the image's
 *                v-th target (1-based); otherwise n_masks >= nt and masks[t] is target row t's mask.  Sizes other than
 *                (mh, mw) are read through nearest-neighbour downsampling (F.interpolate(mode="nearest"))
 *   out_loss   : fp32[5] = [loss*bs, lbox, lseg, lobj, lcls]
 *   grad[l]    : optional, as in y5_loss_fwd_bwd_scaled (mask-coefficient columns included)
 *   grad_proto : optional, same dtype and strides as proto: d(out_loss[0] * upstream)/dproto, every element written
 * Only pixels inside a match's crop are visited.  The loss and grad_proto are deterministic.  The workspace (256-byte
 * aligned) is the detection loss's followed by the segmentation scratch; y5_loss_read_targets works on it too.
 * ------------------------------------------------------------------------------------------------------------- */
int64_t y5_seg_loss_workspace_bytes(const y5_loss_params* p);
int y5_seg_loss_fwd_bwd_scaled(const y5_loss_params* p, const void* const* pl, const float* targets, const float* anchors,
                               const void* proto, int32_t proto_dtype, int64_t ps_b, int64_t ps_k, int64_t ps_y, int64_t ps_x,
                               int32_t nm, int32_t mh, int32_t mw, const float* masks, int32_t n_masks, int32_t gt_h,
                               int32_t gt_w, int32_t overlap, float* out_loss, void* const* grad, void* grad_proto,
                               const float* grad_scale_dev, void* workspace, int64_t workspace_bytes, void* stream);
/* one level's tidx (int64) and xywhn (fp32 x4) of the last y5_seg_loss_fwd_bwd_scaled on this workspace (synchronises) */
int y5_seg_loss_read_targets(const y5_loss_params* p, const void* workspace, int32_t level, int64_t* tidx_host,
                             float* xywhn_host, int32_t* count_host, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Training-mode Conv = SiLU(BN(conv(x)))  (reference models/common.py:86-88; gradients of the same).
 * Forward:   y = conv(x, W)            -> y5_conv_bn_silu_fwd with act = Y5_ACT_NONE and a zero bias (same kernel)
 *            column sums of y          -> y5_bn_stats
 *            z = act(bn(y))            -> y5_bn_act_fwd    (derives mean/invstd, updates running_mean / running_var)
 * Backward:  dy, dgamma, dbeta         -> y5_bn_act_bwd
 *            dW                        -> y5_conv_wgrad    (wgmma, MN-major operands straight from NHWC)
 *            dx = conv(dy, W^T flipped)-> y5_conv_bn_silu_fwd again on transposed/flipped packed weights (stride-2
 *                                         layers first expand dy with y5_zero_stuff2x); `residual` = dx accumulates.
 * Detect.m[i] (models/yolo.py:97) has a bias and no BN: its bias gradient is y5_col_sum(dy).
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct y5_wgrad_desc {
    const void* in;       /* x view, NHWC: element (n,y,x,c) at ((n*in_h + y)*in_w + x)*in_pitch + c */
    int32_t in_pitch;
    int32_t batch, in_h, in_w, in_c;
    const void* dout;     /* dy view [batch*Ho*Wo][out_c], row pitch dout_pitch elements */
    int32_t dout_pitch;
    int32_t out_c;
    float* dweight;       /* fp32 [out_c][ksize][ksize][in_c] (KRSC); zeroed by the call unless accumulate != 0 */
    int32_t ksize, stride, pad;
    int32_t dtype;        /* Y5_F16 | Y5_BF16 (x and dy) */
    int32_t accumulate;
    int32_t reserved;
    /* optional, as in y5_conv_desc: kw != 0 -> filter is ksize x kw with horizontal padding pad_w (dweight is
     * [out_c][ksize][kw][in_c]); non-zero strides (elements) describe a general NHWC view, e.g. overlapping "wide pixels" */
    int32_t kw, pad_w;
    int64_t in_x_stride, in_y_stride, in_n_stride;
} y5_wgrad_desc;
int y5_conv_wgrad(const y5_wgrad_desc* d, void* stream);

/* Training BatchNorm + activation, in five passes:
 *   forward:  y5_bn_stats (column sums) -> y5_bn_act_fwd (normalise + activate)
 *   backward: y5_bn_act_bwd (reduce + apply), or, split for SyncBatchNorm, y5_bn_act_bwd_reduce -> y5_bn_act_bwd_apply
 * act: Y5_ACT_NONE | Y5_ACT_SILU | Y5_ACT_LEAKY; `slope` is the negative slope of Y5_ACT_LEAKY (finite; 0 = ReLU) and is
 * ignored otherwise.  LeakyReLU, with t = bn(y) rounded to the activation dtype:
 *   forward:  z = round(t > 0 ? t : slope * t)                       (fp32 product; + residual as below)
 *   backward: du = round(t > 0 ? dz : dz * slope)                    (torch's leaky_relu_backward), parked in dy like SiLU's
 * SyncBatchNorm (torch.nn.SyncBatchNorm in training under torch.distributed) adds the column sums of every rank with the
 * caller's SUM all-reduce between passes.  Its forward workspace is 2 * channels + 1 doubles, ZERO on entry; slot 2 * channels
 * is the row count:
 *   forward:  y5_bn_stats(count = ws + 2C) -> all-reduce ws[0 .. 2C] -> y5_bn_act_fwd(sums = ws, count = ws + 2C)
 *   backward: y5_bn_act_bwd_reduce -> all-reduce ws[0 .. 2C) -> y5_bn_act_bwd_apply(count = the forward's N)
 * `count` points at one fp64 row count, or is NULL for plain BatchNorm, where `rows` is the whole batch (y5_bn_act_bwd_apply
 * requires it; y5_bn_act_fwd takes it only with `sums`).  y5_bn_stats adds `rows` to *count; y5_bn_act_fwd and
 * y5_bn_act_bwd_apply divide by the N it holds instead of `rows`, and y5_bn_act_fwd's running_var takes the unbiased factor
 * N / (N - 1).  Without the all-reduce, the SyncBatchNorm passes compute exactly what the plain ones compute. */
/* workspace of y5_bn_stats / y5_bn_act_bwd / y5_col_sum: 2 * channels doubles.  For y5_bn_stats and y5_bn_act_bwd it
 * must be ZERO on entry and is left dirty (callers carve it from one arena cleared once per step); y5_col_sum clears
 * its own. */
int64_t y5_bn_workspace_bytes(int32_t channels);
/* per-channel sum and sum of squares of a [rows][channels] view, accumulated into workspace (fp64) */
int y5_bn_stats(const void* y, int32_t pitch, int64_t rows, int32_t channels, int32_t dtype, void* workspace,
                double* count, void* stream);
/* z = act(gamma * (y - mean) * invstd + beta); z may be a channel-slice view.
 * sums != NULL (training): mean / invstd (biased variance + eps) are first derived from the y5_bn_stats workspace and
 * WRITTEN to mean / invstd, and running_mean / running_var (nullable) are updated like nn.BatchNorm2d does (momentum,
 * unbiased variance).  sums == NULL (eval): mean / invstd are inputs.  residual != NULL adds a view of the same shape
 * after the activation (Bottleneck shortcut, models/common.py:181); its gradient is dz itself. */
int y5_bn_act_fwd(const void* y, int32_t y_pitch, void* z, int32_t z_pitch, int64_t rows, int32_t channels,
                  int32_t dtype, float* mean, float* invstd, const float* gamma, const float* beta, int32_t act, float slope,
                  const void* sums, const void* count, float eps, float momentum, float* running_mean, float* running_var,
                  const void* residual, int32_t res_pitch, void* stream);
/* given dz: dy (gradient w.r.t. the conv output), dgamma, dbeta (fp32, overwritten).  Two launches: the reduce pass forms
 * du = dz * act'(bn(y)) and its two column sums and, for Y5_ACT_SILU / Y5_ACT_LEAKY, parks du in the dy buffer; the apply
 * pass turns it into dy in place.  dy may alias dz (every element is read before it is written) but not y. */
int y5_bn_act_bwd(const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                  int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd,
                  const float* gamma, const float* beta, int32_t act, float slope, float* dgamma, float* dbeta,
                  void* workspace, void* stream);
/* the reduce pass of y5_bn_act_bwd: the column sums into the workspace, THIS rank's dgamma / dbeta from them and, for
 * Y5_ACT_SILU / Y5_ACT_LEAKY, du left in dy */
int y5_bn_act_bwd_reduce(const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                         int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd,
                         const float* gamma, const float* beta, int32_t act, float slope, float* dgamma, float* dbeta,
                         void* workspace, void* stream);
/* the apply pass of y5_bn_act_bwd with the all-reduced `sums` and `count` (required); dgamma / dbeta untouched.  It only
 * reads the parked du, so it takes no slope. */
int y5_bn_act_bwd_apply(const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                        int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd,
                        const float* gamma, int32_t act, const void* sums, const void* count, void* stream);
/* out[c] = sum over rows of y[row][c] (fp32) */
int y5_col_sum(const void* y, int32_t pitch, int64_t rows, int32_t channels, int32_t dtype, float* out, void* workspace,
               void* stream);
/* OIHW master weights (Y5_F32 | Y5_F16 | Y5_BF16) -> K-major packings in `dtype` for y5_conv_bn_silu_fwd, either may be
 * NULL:  fwd [out_c][k][k][in_c_pad] = w[o][i][r][s]  and  dgrad [in_c][k][k][out_c_pad] = w[o][i][k-1-r][k-1-s]
 * (padding channels zero; pads = channel counts rounded up to the block_k y5_conv_pick returns). */
int y5_weight_pack(const void* w, int32_t w_dtype, int32_t out_c, int32_t in_c, int32_t ksize, void* fwd, int32_t in_c_pad,
                   void* dgrad, int32_t out_c_pad, int32_t dtype, void* stream);
/* The same for every filter of a model in ONE launch (the training step re-packs its fp32 master weights once per forward):
 * `items` (device memory) describes the filters exactly like the arguments of y5_weight_pack; block b of the launch converts
 * elements [chunk_index[b] * y5_weight_pack_chunk_elems(), ...) of the concatenated [fwd | dgrad] packing of item chunk_item[b]
 * (both arrays in device memory, built once per model by the caller). */
typedef struct y5_pack_item {
    const void* w;
    void* fwd;
    void* dgrad;
    int32_t w_dtype;
    int32_t out_c, in_c, ksize;
    int32_t in_c_pad, out_c_pad;
} y5_pack_item;
int32_t y5_weight_pack_chunk_elems(void);
int y5_weight_pack_multi(const y5_pack_item* items, const int32_t* chunk_item, const int32_t* chunk_index, int32_t n_chunks,
                         int32_t dtype, void* stream);
/* backward of y5_upsample2x: dx[n,i,j,:] = dy[n,2i,2j,:] + dy[n,2i,2j+1,:] + dy[n,2i+1,2j,:] + dy[n,2i+1,2j+1,:] */
int y5_upsample2x_bwd(const void* dy, int32_t dy_pitch, void* dx, int32_t dx_pitch, int32_t batch, int32_t h, int32_t w,
                      int32_t c, int32_t dtype, void* stream);
/* backward of y5_sppf_pool + the concat of SPPF (models/common.py:338-340): cat = [a, m(a), m(m(a)), m(m(m(a)))] as 4
 * channel slices of c channels (the forward's buffer), dcat its gradient; writes da.  Arg-max ties resolve to the
 * first maximum in row-major window order, as torch's max_pool2d backward does.  workspace: 3*B*h*w*c floats. */
int64_t y5_sppf_bwd_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t c);
int y5_sppf_pool_bwd(const void* cat, int32_t cat_pitch, const void* dcat, int32_t dcat_pitch, void* da, int32_t da_pitch,
                     int32_t batch, int32_t h, int32_t w, int32_t c, int32_t ksize, int32_t dtype, void* workspace,
                     void* stream);
/* Max-pools of the YOLOv3 models over NHWC views (x: h x w, c channels), dtype Y5_F16 | Y5_BF16 | Y5_F32:
 *   Y5_POOL_K2S2       nn.MaxPool2d(2, 2, 0): y is (h/2) x (w/2)
 *   Y5_POOL_K2S1_ZPAD  nn.ZeroPad2d((0, 1, 0, 1)) then nn.MaxPool2d(2, 1, 0): y is h x w; the pad cells hold 0
 * A NaN in a window makes its maximum NaN.  The backward writes dx: each window's gradient goes to its first maximum in
 * row-major window order (a NaN takes it from earlier cells), as torch's max_pool2d backward does; a window whose maximum
 * is a pad cell routes nowhere.  Views are 16-byte aligned, c and pitches multiples of 8 (Y5_E_INVALID / Y5_E_UNSUPPORTED). */
#define Y5_POOL_K2S2 0
#define Y5_POOL_K2S1_ZPAD 1
int y5_maxpool2d(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                 int32_t mode, int32_t dtype, void* stream);
int y5_maxpool2d_bwd(const void* x, int32_t x_pitch, const void* dy, int32_t dy_pitch, void* dx, int32_t dx_pitch, int32_t batch,
                     int32_t h, int32_t w, int32_t c, int32_t mode, int32_t dtype, void* stream);
/* backward of SPP's pools + concat (models/common.py SPP): cat = [a, mp_k(a), mp_2k-1(a), mp_3k-2(a)] (the y5_sppf_pool
 * buffer), dcat its gradient (4 slices of c channels).  da = dcat[0] + each window's gradient routed to the first maximum
 * of that window of `a` (torch's tie rule, unlike y5_sppf_pool_bwd's chain through the intermediate pools), summed in fp32
 * and rounded once.  dtype Y5_F16 | Y5_BF16 | Y5_F32; workspace: y5_spp_bwd_workspace_bytes, 16-byte aligned. */
int64_t y5_spp_bwd_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t c);
int y5_spp_pool_bwd(const void* a, int32_t a_pitch, const void* dcat, int32_t dcat_pitch, void* da, int32_t da_pitch,
                    int32_t batch, int32_t h, int32_t w, int32_t c, int32_t ksize, int32_t dtype, void* workspace, void* stream);
/* y[n, 2i, 2j, :] = x[n, i, j, :], other pixels of the (2h, 2w) output zero */
int y5_zero_stuff2x(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w,
                    int32_t c, int32_t dtype, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * The callers either side of the hot path (SURVEY.md section 8f), batched on the device, no host synchronisation.
 * ------------------------------------------------------------------------------------------------------------------ */
/* Pre-processing: letterbox (utils/augmentations.py:85-115: cv2.resize INTER_LINEAR to (new_w,new_h), constant border) +
 * BGR->RGB + HWC->CHW (utils/dataloaders.py:354-357) + uint8 -> float /255 (detect.py:205-208, val.py:259-262,
 * models/common.py:924-926) for a batch of device-resident uint8 HWC images of different sizes.  The resize is OpenCV's
 * fixed-point bilinear kernel restated bit for bit (oracle/pre_ref.py, pinned against the installed cv2).  The geometry
 * (new_w/new_h/top/left) is computed by the caller exactly as the reference's letterbox() does. */
typedef struct y5_letterbox_image {
    const void* data;       /* uint8 HWC, 3 channels, device memory */
    int32_t src_h, src_w;
    int32_t row_bytes;      /* bytes between source rows (>= 3*src_w) */
    int32_t new_h, new_w;   /* size after cv2.resize ("new_unpad") */
    int32_t top, left;      /* border offsets inside the (out_h, out_w) canvas */
} y5_letterbox_image;
int y5_letterbox_max_images(void); /* descriptors are consumed in groups of this many per launch */
/* out: out_dtype Y5_U8 -> (n,3,out_h,out_w) bytes (what the dataloader yields); Y5_F16/BF16/F32 -> the same /255;
 * s2d != 0 (fp16/bf16 only) -> the stem's 2x2 space-to-depth cells, layout and out_row_px/out_x_off as in y5_stem_s2d.
 * `images` is a HOST array (copied into the launch parameters). */
int y5_letterbox(const y5_letterbox_image* images, int32_t n_images, int32_t out_h, int32_t out_w, int32_t swap_rb,
                 int32_t pad_value, void* out, int32_t out_dtype, int32_t s2d, int32_t out_row_px, int32_t out_x_off,
                 void* stream);

/* Validation batch (utils/dataloaders.py:711-766, augment=False): load_image's resize of each ORIGINAL image to
 * (res_h, res_w) = (ceil(h0 r), ceil(w0 r)) -- Y5_VAL_AREA (cv2 INTER_AREA, r < 1), Y5_VAL_LINEAR (cv2 INTER_LINEAR,
 * r > 1) or Y5_VAL_COPY (r == 1) -- then letterbox(auto=False, scaleup=False) into the (out_h, out_w) canvas with
 * border 114, CHW with RGB order.  Both resizes are OpenCV's arithmetic restated bit for bit (oracle/val_load_ref.py).
 * When letterbox resizes again ((new_h, new_w) != (res_h, res_w)) the load_image result is written HWC BGR to the
 * image's `scratch` (res_h * res_w * 3 bytes, DEVICE) and y5_letterbox takes it from there; otherwise scratch is unused
 * and the image sits at (top, left) unchanged.  out: (n, 3, out_h, out_w) Y5_U8, or Y5_F16 | Y5_BF16 | Y5_F32 as
 * float32(v) * float32(1 / 255) rounded once (what `im.half() / 255` computes on a CUDA tensor).  `images` is a HOST
 * array; sources and out are DEVICE memory.  No allocation and no host synchronisation. */
#define Y5_VAL_COPY 0
#define Y5_VAL_LINEAR 1
#define Y5_VAL_AREA 2
struct y5_val_image {
    const void* data;       /* the original image: uint8 HWC BGR, 3 channels */
    void* scratch;          /* (res_h, res_w, 3) uint8 when new != res, else NULL */
    int32_t src_h, src_w;
    int32_t row_bytes;      /* bytes between source rows (>= 3 * src_w) */
    int32_t res_h, res_w;   /* load_image's size */
    int32_t interp;         /* Y5_VAL_* */
    int32_t new_h, new_w;   /* letterbox's new_unpad */
    int32_t top, left;      /* letterbox's border offsets inside the canvas */
};
typedef struct y5_val_image y5_val_image;
int y5_val_letterbox(const y5_val_image* images, int32_t n_images, int32_t out_h, int32_t out_w, void* out, int32_t out_dtype,
                     void* stream);

/* Classification batch (utils/augmentations.py classify_transforms, utils/dataloaders.py:949-985 without Albumentations):
 * CenterCrop's cv2.resize INTER_LINEAR of each image's center m x m square to (out_h, out_w), then ToTensor (BGR -> RGB,
 * CHW, float32 v / 255 as a true division) and Normalize ((v - mean[c]) / std[c] in float32).  `data` holds only the
 * square: m rows of `row_bytes` bytes, uint8 BGR.  out: (n, 3, out_h, out_w) Y5_F32, or Y5_F16 | Y5_BF16 as that float32
 * value rounded once.  `images` is a DEVICE array of n descriptors (so one launch takes any batch size); the descriptors are
 * the caller's to get right (an image with side <= 0 or row_bytes < 3 * side is skipped).  mean, std: 3 HOST float32 values
 * each, in RGB order.  No allocation and no host synchronisation. */
struct y5_cls_image {
    const void* data;   /* the center square: uint8 HWC BGR, 3 channels, DEVICE */
    int32_t side;       /* m = min(h, w) of the original image */
    int32_t row_bytes;  /* bytes between rows (>= 3 * side) */
};
typedef struct y5_cls_image y5_cls_image;
int y5_cls_batch(const y5_cls_image* images, int32_t n_images, int32_t out_h, int32_t out_w, const float* mean, const float* std, void* out,
                 int32_t out_dtype, void* stream);

/* process_mask (utils/segment/general.py:25-52, crop_mask :10-22): for detection i of image img_index[i] (NULL = image 0):
 * sigmoid(coef_i . protos[img]) at mask resolution, zeroed outside the box scaled by (mw/in_w, mh/in_h), optionally
 * bilinearly up-sampled (align_corners=False) to (in_h,in_w), thresholded at 0.5.
 *   mode 0: process_mask(upsample=False) -> (n, mh, mw);  mode 1: process_mask(upsample=True) -> (n, in_h, in_w);
 *   mode 2: process_mask_native (:55-76): no low-resolution crop, the prototype window [top, left, height, width] (`window`,
 *           HOST array of 4 ints) is up-sampled to (in_h, in_w) and cropped to the un-scaled boxes -> (n, in_h, in_w)
 *   protos (batch, c, mh, mw) NCHW Y5_F16|Y5_BF16|Y5_F32 (read as float, like `protos.float()`); coef rows of `coef_stride`
 *   floats (may point at column 6 of the NMS rows); boxes rows of `box_stride` floats, xyxy in network-input pixels;
 *   out Y5_F32 {0,1} (the reference's `masks.gt_(0.5)`) or Y5_U8.
 * Detections of the same image must be adjacent.  workspace: y5_process_mask_workspace_bytes (modes 1, 2). */
int64_t y5_process_mask_workspace_bytes(int32_t n, int32_t mh, int32_t mw, int32_t mode);
int y5_process_mask(const void* protos, int32_t proto_dtype, int32_t batch, int32_t c, int32_t mh, int32_t mw, const float* coef,
                    int32_t coef_stride, const float* boxes, int32_t box_stride, const int32_t* img_index, int32_t n,
                    int32_t in_h, int32_t in_w, int32_t mode, const int32_t* window, void* out, int32_t out_dtype,
                    void* workspace, int64_t workspace_bytes, void* stream);
/* crop_mask (utils/segment/general.py:10-22): out = masks * [box contains the pixel]; masks/out (n,h,w) fp32 */
int y5_crop_mask(const float* masks, const float* boxes, int32_t box_stride, int32_t n, int32_t h, int32_t w, float* out,
                 void* stream);

/* scale_boxes + clip_boxes (utils/general.py:613-626), in place on rows of `row_stride` floats (xyxy first).
 * meta: per image 5 floats [gain, pad_x, pad_y, w0, h0] (device).  Image of row i = img_index[i], or i / rows_per_image
 * when img_index is NULL (then `count`, if given, limits each image to its first count[img] rows: the padded layout
 * y5_nms_batched produces), or 0 when both are absent. */
int y5_scale_boxes(float* boxes, int32_t row_stride, int64_t n_rows, const int32_t* img_index, int32_t rows_per_image,
                   const int32_t* count, const float* meta, void* stream);
/* val.py:303-306 for the whole batch: targets (nt,6) [img, cls, cx, cy, w, h] in network-input pixels ->
 * out (nt,6) [img, cls, x1, y1, x2, y2] in native pixels (xywh2xyxy, then scale_boxes with the image's meta). */
int y5_labels_native(const float* targets, int32_t nt, const float* meta, float* out, void* stream);
/* process_batch (utils/metrics.py:224-265, box branch) for every image of a batch in one launch:
 *   det (batch, max_det, row_stride>=6) fp32 rows [x1,y1,x2,y2,conf,cls,...] in native pixels (image b at det + b*img_stride),
 *   count[b] valid rows (NULL = max_det); labels (nt,6) [img, cls, x1,y1,x2,y2] in any order; iouv (niou) thresholds;
 *   correct (batch, max_det, niou) uint8: the reference's boolean matrix (rows >= count[b] are 0).  Bit-exact. */
int y5_match_batch(const float* det, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t batch,
                   int32_t max_det, const float* labels, int32_t nt, const float* iouv, int32_t niou, float eps,
                   uint8_t* correct, void* stream);
/* ConfusionMatrix.process_batch (utils/metrics.py:139-183) for every image of a batch in one launch, added into `matrix`.
 *   det / img_stride / row_stride / count as y5_match_batch (rows [x1,y1,x2,y2,conf,cls,...] in native pixels, row_stride >= 6);
 *   labels (nt,6) [img, cls, x1,y1,x2,y2] in target order; matrix (nc+1, nc+1) int64, row = predicted class, column = true
 *   class, index nc = background.  Per image: detections with conf > conf_thres (fp32 compare) are kept; a (label, kept
 *   detection) pair is a candidate when box_iou > iou_thres; each detection keeps its best candidate label (first label on
 *   equal IoU), then each label keeps, among the detections whose best it is, the one of highest IoU (first detection on
 *   equal IoU).  A matched label adds 1 at [det class, label class], an unmatched one at [nc, label class]; when the image has
 *   a match, every kept detection no label kept adds 1 at [det class, nc].  An image without rows counts its labels as
 *   background, one without labels counts nothing (val.py's per-image branching gives these same counts).  Classes are
 *   `.int()` of the value; one outside [0, nc) writes nothing and ORs 1 (a label's) or 2 (a detection's) into `*error`
 *   (int32, device).  Integer atomics: repeatable bit for bit.  max_det <= 4096, nc <= 32768. */
int y5_confusion_batch(const float* det, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t batch,
                       int32_t max_det, const float* labels, int32_t nt, int32_t nc, float conf_thres, float iou_thres, float eps,
                       int64_t* matrix, int32_t* error, void* stream);

/* Mask IoU of segment/val.py (utils/metrics.py:239-265 process_batch(masks=True); ultralytics' mask_iou) as a 1-bit GEMM.
 * Bit rows: an (h, w) mask is y5_mask_row_words(h, w) uint32 words, pixel p = y*w + x at bit p%32 of word p/32, zero bits
 * up to a multiple of 256 pixels.  y5_mask_row_words returns Y5_E_UNSUPPORTED when h*w > 2^23 (beyond that the reference's
 * fp32 pixel sums stop being exact).
 * label_index (device, batch + 1 + 2*nt int32, written by y5_mask_pack whenever it is given, nt = 0 included): [0..batch] the first row
 * of each image's labels (image b owns rows [li[b], li[b+1]) in target order), then for every row its target index, then
 * its image (-1: the target's image column is not an integer in [0, batch); such rows follow li[batch]). */
int32_t y5_mask_row_words(int32_t h, int32_t w);
/* Masks -> bit rows (out_h, out_w) + popcount (n_rows int32), reading `src` (contiguous planes of src_h*src_w, Y5_U8 (also
 * bool) | Y5_F32 | Y5_F16 | Y5_BF16).  One block per row; an overlap index plane is read once per label of its image.
 *   overlap == 0, label_index NULL : row r = plane r (direct 0/1 masks)
 *   overlap == 0, label_index set  : rows of the nt = n_rows targets grouped by image: row = plane row_target (segment/val.py
 *                                    `masks[targets[:, 0] == si]`, so src holds nt planes)
 *   overlap != 0, label_index NULL : row k = (plane 0 == k + 1), k < n_rows (one image's index mask, `gt == arange(nl) + 1`)
 *   overlap != 0, label_index set  : row of label k of image b = (plane b == k + 1) (src holds batch planes)
 * With label_index, `batch` images and target_img (device: the image column of the (nt, target_stride) fp32 targets, may be
 * NULL when nt == 0) lay out the label rows first.  When (src_h, src_w) != (out_h, out_w) each
 * row's values (the 0/1 indicators in overlap mode) are resized as F.interpolate(bilinear, align_corners=False) and kept
 * where > 0.5.  Direct values that are not 0 or 1 and enter unresized are added to *nonbinary (device int32). */
int y5_mask_pack(const void* src, int32_t src_dtype, int32_t src_h, int32_t src_w, int32_t overlap, const float* target_img,
                 int32_t target_stride, int32_t batch, int32_t n_rows, int32_t out_h, int32_t out_w, int32_t* label_index,
                 uint32_t* bits, int32_t* popcount, int32_t* nonbinary, void* stream);
/* iou[(l) * rows_per_image + d] = inter / (|gt_l| + |pred_d| - inter + eps) for images img0..img0+n_img-1: labels l of image b
 * from label_index, predictions d < count[b] (NULL: all) at pred rows (b - img0) * rows_per_image + d.  label_index NULL: one
 * image, labels 0..n_gt-1 (the single-pair mask_iou(gt, pred) -> (n_gt, rows_per_image)).  `words` = y5_mask_row_words. */
int y5_mask_iou(const uint32_t* gt_bits, const int32_t* gt_pop, const int32_t* label_index, int32_t n_gt, const uint32_t* pred_bits,
                const int32_t* pred_pop, const int32_t* count, int32_t img0, int32_t n_img, int32_t rows_per_image, int32_t words,
                float eps, float* iou, void* stream);
/* process_batch(masks=True)'s matching (utils/metrics.py:255-264) for every image of a batch, reading the IoU matrix of
 * y5_mask_iou (rows_per_image = max_det): det / count / correct as y5_match_batch; label l's class at
 * label_cls[target(l) * cls_stride] (target(l) from label_index, or l when label_index is NULL and batch == 1). */
int y5_mask_match_batch(const float* det, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t batch, int32_t max_det,
                        const float* label_cls, int32_t cls_stride, const int32_t* label_index, int32_t nt, const float* iou,
                        const float* iouv, int32_t niou, uint8_t* correct, void* stream);

/* Fused optimizer step (train.py:413-421): un-scale + clip_grad_norm_ + SGD(momentum, nesterov) over parameter groups
 * (utils/torch_utils.py:256-289) + optimizer.zero_grad + ModelEMA.update (utils/torch_utils.py:359-368) in two
 * multi-tensor launches.  All tensors fp32.  `table`, `chunk_*`, `hyper`, `partial` are DEVICE arrays owned by the caller:
 *   table[t]            one entry per tensor (buffers take part in the EMA only: grad = mom = NULL)
 *   chunk_tensor/index  block c handles elements [chunk_index[c]*y5_opt_chunk_elems(), +y5_opt_chunk_elems()) of tensor chunk_tensor[c]
 *   hyper               floats: [Y5_OPT_INV_SCALE] 1/loss scale, [Y5_OPT_MAX_NORM] clip norm (<= 0: off), [Y5_OPT_EMA_DECAY],
 *                       [Y5_OPT_EMA_TAU], [Y5_OPT_EMA_UPDATES] counter (advanced by the call when do_ema),
 *                       [Y5_OPT_OUT_NORM] total gradient norm (written), [Y5_OPT_OUT_SKIPPED] 1 if a non-finite gradient
 *                       made the step skip (written), then per group g at Y5_OPT_GROUPS + 4g: lr, momentum, weight_decay, nesterov
 *   partial             2 * n_chunks floats of scratch */
typedef struct y5_opt_tensor {
    void* param;
    void* grad;
    void* mom;
    void* ema;
    int64_t numel;
    int32_t group;
    int32_t reserved;
} y5_opt_tensor;
#define Y5_OPT_INV_SCALE 0
#define Y5_OPT_MAX_NORM 1
#define Y5_OPT_EMA_DECAY 2
#define Y5_OPT_EMA_TAU 3
#define Y5_OPT_EMA_UPDATES 4
#define Y5_OPT_OUT_NORM 5
#define Y5_OPT_OUT_SKIPPED 6
#define Y5_OPT_GROUPS 8
int32_t y5_opt_chunk_elems(void);
int y5_opt_step(const y5_opt_tensor* table, const int32_t* chunk_tensor, const int32_t* chunk_index, int32_t n_chunks,
                float* hyper, float* partial, int32_t do_step, int32_t do_ema, int32_t zero_grad, void* stream);

/* The same step with Adam / AdamW (utils/torch_utils.py:276-279: torch.optim.Adam(betas=(momentum, 0.999)) or
 * AdamW(weight_decay=0) plus the two decay groups) in three launches: y5_opt_step's gradient-norm pass, the update, and a tail
 * that advances the step counters and the EMA counter.  Per parameter with a gradient, after un-scaling and clipping:
 *   Adam: g += wd*p   AdamW: p *= 1 - lr*wd;   m = lerp(m, g, 1 - b1);  v = v*b2 + (1 - b2)*g*g;  step += 1;
 *   p += -(lr / (1 - b1^step)) * m / (sqrt(v) / sqrt(1 - b2^step) + eps)
 * with torch.optim.Adam's order of operations; 1 - b1, 1 - b2, the powers and the two corrections are computed in double and
 * rounded to fp32 where torch rounds its Python scalars.  A non-finite gradient skips the update (p, m, v and steps unchanged).
 *   table, chunk_*, hyper, partial  as y5_opt_step (do_step is implied); the per-group block of `hyper` is unused.  table[t].mom
 *                       points at tensor t's exp_avg, its exp_avg_sq is at exp_avg + sq_offset elements.
 *   n_tensors           entries of `table`
 *   group_hyper         DEVICE doubles (a separate argument, so 8-byte aligned by construction): per group g at
 *                       Y5_ADAM_STRIDE * g: lr, beta1, beta2, eps, weight_decay, decoupled (!= 0: AdamW)
 *   steps               DEVICE floats, steps[t] = step count of table entry t (torch's fp32 state["step"]); it advances
 *                       only for entries with a gradient and mom on a step that was not skipped */
#define Y5_ADAM_LR 0
#define Y5_ADAM_BETA1 1
#define Y5_ADAM_BETA2 2
#define Y5_ADAM_EPS 3
#define Y5_ADAM_WEIGHT_DECAY 4
#define Y5_ADAM_DECOUPLED 5
#define Y5_ADAM_STRIDE 8
int y5_adam_step(const y5_opt_tensor* table, int32_t n_tensors, const int32_t* chunk_tensor, const int32_t* chunk_index, int32_t n_chunks,
                 float* hyper, const double* group_hyper, int64_t sq_offset, float* steps, float* partial, int32_t do_ema,
                 int32_t zero_grad, void* stream);

/* Data-parallel gradient exchange, device half (utils/torch_utils.py:61-70 smart_DDP / train.py:404-414): copy every gradient
 * of `table` (entries with mom != NULL; a NULL grad contributes zeros) into ONE contiguous fp32 arena in a single launch, so the
 * all-reduce is one NCCL call over the arena and y5_opt_step reads the averaged gradients from it (a second table whose grad
 * pointers are arena + arena_offset[t]).  arena_offset[t]: element offset of tensor t, a multiple of 4; arena 16-byte aligned.
 * present[t] = 1.0 / 0.0: tensor t had a gradient on this rank (callers place `present` right behind the arena so the same
 * all-reduce averages it); y5_grad_bind then rewrites the arena table's gradient pointers -- NULL where present[t] == 0 on every
 * rank -- so the update skips such parameters like the single-process step does. */
int y5_grad_pack(const y5_opt_tensor* table, const int32_t* chunk_tensor, const int32_t* chunk_index, int32_t n_chunks,
                 const int64_t* arena_offset, float* arena, float* present, void* stream);
int y5_grad_bind(y5_opt_tensor* arena_table, int32_t n_tensors, const int64_t* arena_offset, float* arena, const float* present,
                 void* stream);

/* Fold eval-mode BatchNorm into a conv and pack it for y5_conv_bn_silu_fwd in ONE launch (utils/torch_utils.py:224-254):
 *   packed[o][r][s][i_pad] = w[o][i][r][s] * gamma[o] / sqrt(var[o] + eps)   (activation dtype, zero padded)
 *   bias_out[o]            = beta[o] + (conv_bias[o] - mean[o]) * gamma[o] / sqrt(var[o] + eps)   (fp32)
 * gamma == NULL: no BatchNorm (already fused conv): packed = w, bias_out = conv_bias (or 0).  w: OIHW Y5_F32|F16|BF16;
 * BN tensors fp32 or the weight dtype (`bn_dtype`).  out_c_pad >= out_c rows are written (extra rows zero, bias 0). */
int y5_fold_pack(const void* w, int32_t w_dtype, int32_t out_c, int32_t in_c, int32_t kh, int32_t kw, const void* conv_bias,
                 const void* gamma, const void* beta, const void* mean, const void* var, int32_t bn_dtype, float eps,
                 void* packed, int32_t in_c_pad, int32_t out_c_pad, float* bias_out, int32_t dtype, void* stream);

/* Training augmentation (utils/dataloaders.py:696-855 __getitem__ / load_mosaic, utils/augmentations.py:69-82 augment_hsv,
 * :118-197 random_perspective (affine), :225-233 mixup) for a batch, byte-exact with the reference's OpenCV arithmetic
 * (oracle/aug_ref.py).  The host draws every random number; the device table below carries the result.
 * A "mosaic" is a virtual canvas (canvas_w x canvas_h, 114 outside its tiles) made of up to 4 tiles: canvas pixel
 * (x, y) inside tile t's rectangle [x1a, x2a) x [y1a, y2a) reads src + (y + dy) * row_bytes + (x + dx) * pixel_stride
 * + channel * channel_stride (BGR channel order).  An output image is warp(mosaic 0), or with mixup
 * trunc(warp(mosaic 0) * mix_r + warp(mosaic 1) * (1 - mix_r)), then the three HSV LUTs, then the flips.
 * (Declared as struct + typedef; tests/test_augment_cpu.py checks their layout against the ctypes mirrors.) */
struct y5_aug_tile {
    const void* src;                /* uint8, device memory */
    int32_t row_bytes, pixel_stride, channel_stride;
    int32_t x1a, y1a, x2a, y2a;     /* rectangle on the canvas */
    int32_t dx, dy;                 /* source pixel = canvas pixel + (dx, dy) */
    int32_t reserved;
};
typedef struct y5_aug_tile y5_aug_tile;
struct y5_aug_image {
    double inv_m[2][6];     /* cv2.invertAffineTransform(M[:2]) per mosaic, row-major */
    double m[2][6];         /* M[:2] per mosaic (labels) */
    double mix_r;           /* mixup ratio r, used when n_mosaic == 2 */
    float scale[2];         /* random_perspective's scale draw per mosaic (box_candidates) */
    float clip_max;         /* load_mosaic's label clip bound 2*s (labels with Y5_AUG_CLIP) */
    int32_t n_mosaic;       /* 1, or 2 with mixup */
    int32_t n_tiles[2];     /* tiles [0, n_tiles[0]) belong to mosaic 0, [4, 4 + n_tiles[1]) to mosaic 1 */
    int32_t canvas_w, canvas_h;
    int32_t warp[2];        /* 0: M == I, the canvas is the image (random_perspective skips cv2.warpAffine) */
    int32_t hsv, flipud, fliplr;
    int32_t reserved;
    y5_aug_tile tiles[8];
    uint8_t lut[3][256];    /* hue, saturation, value LUTs (augment_hsv), used when hsv != 0 */
};
typedef struct y5_aug_image y5_aug_image;
/* One input label row and its path to the output.  flags: Y5_AUG_CLIP clips the xyxy box to [0, clip_max] (load_mosaic);
 * Y5_AUG_IN_XYXY: (x, y, w, h) already hold pixel x1, y1, x2, y2 (tile_w ... pad_h unused); Y5_AUG_OUT_XYXY: write the
 * warped pixel xyxy box (random_perspective's return) instead of xyxy2xywhn(clip=True, eps=1e-3) + flips. */
#define Y5_AUG_CLIP 1
#define Y5_AUG_IN_XYXY 2
#define Y5_AUG_OUT_XYXY 4
struct y5_aug_label {
    float cls, x, y, w, h;                  /* normalised xywh, float32 as the dataset stores it */
    float tile_w, tile_h, pad_w, pad_h;     /* xywhn2xyxy's w, h, padw, padh, already rounded to float32 */
    int32_t image, mosaic, flags;
};
typedef struct y5_aug_label y5_aug_label;
/* out: (n, 3, out_h, out_w) Y5_U8 | Y5_F16 | Y5_BF16 | Y5_F32 (/255), RGB when swap_rb (BGR otherwise); s2d != 0
 * (fp16/bf16, even sizes) writes the stem's space-to-depth cells instead (layout and out_row_px/out_x_off as in
 * y5_stem_s2d).  hsv_simd_cols: columns [0, hsv_simd_cols) of a row truncate in HSV->BGR, the rest round (cv2's SIMD
 * blocks and scalar tail: out_w - out_w % 32).  `table` is DEVICE memory. */
int y5_aug_gather(const y5_aug_image* table, int32_t n_images, int32_t out_h, int32_t out_w, int32_t hsv_simd_cols, int32_t swap_rb,
                  void* out, int32_t out_dtype, int32_t s2d, int32_t out_row_px, int32_t out_x_off, void* stream);
/* Labels of a batch in input order -> the kept rows, compacted stably, as collate_fn's (nt, 6) float32 [image, cls, box]
 * rows in `targets` (room for n_labels rows); *count (device int32) = nt.  `table` and `labels` are DEVICE memory. */
int y5_aug_labels(const y5_aug_image* table, int32_t n_images, const y5_aug_label* labels, int32_t n_labels, int32_t out_h,
                  int32_t out_w, float* targets, int32_t* count, void* stream);

/* Segmentation training augmentation (utils/segment/dataloaders.py:130-301, utils/segment/augmentations.py:26-91 and
 * ultralytics' polygons2masks[_overlap]), exact with the reference's numpy / OpenCV arithmetic (oracle/seg_aug_ref.py).
 * Images go through y5_aug_gather with the same table; each label row (y5_aug_label, with the xyn2xy parameters in
 * tile_w .. pad_h) has one polygon: n_points normalised float32 (x, y) pairs starting at pair point_offset of `points`.
 * All pointers are DEVICE memory.  Sizes: verts n_labels * Y5_SEG_POINTS * 2 int32, rows n_labels * 6, masks
 * n_labels * (out_h / r) * (out_w / r) bytes. */
#define Y5_SEG_POINTS 1000 /* resample_segments(n=1000) */
#define Y5_SEG_I32 4       /* y5_seg_compose's int32 output (overlap masks of images with more than 255 labels) */
struct y5_aug_segment {
    int32_t point_offset, n_points;
};
typedef struct y5_aug_segment y5_aug_segment;
/* Per label: the resampled, warped polygon as polygon2mask's int32 vertices (verts), keep = box_candidates(area_thr 0.01)
 * of its segment2box box, and its collate_fn row [image, cls, xywhn] (flips applied) in rows.  max_points bounds n_points. */
int y5_seg_warp(const y5_aug_image* table, int32_t n_images, const y5_aug_label* labels, const y5_aug_segment* segments,
                const float* points, int32_t max_points, int32_t n_labels, int32_t out_h, int32_t out_w, int32_t* verts, float* rows,
                int32_t* keep, void* stream);
/* cv2.resize(cv2.fillPoly(zeros(out_h, out_w), [poly], 1), (out_w / r, out_h / r)) for every kept label, unflipped, and
 * its area (sum of the mask).  Polygon i is verts[i * n_verts * 2 ...], n_verts int32 (x, y) vertices (y5_seg_warp's:
 * Y5_SEG_POINTS).  ratio: 1 or 4 (Y5_E_UNSUPPORTED otherwise; out_h, out_w multiples of it). */
int y5_seg_raster(const int32_t* verts, int32_t n_verts, const int32_t* keep, int32_t n_labels, int32_t out_h, int32_t out_w,
                  int32_t ratio, uint8_t* masks, int32_t* areas, void* stream);
/* Image b owns label rows [image_rows[b], image_rows[b + 1]).  Kept labels -> output positions: image order, and within an
 * image label order, or with overlap the order of np.argsort(-areas) on uint64 (zero areas first, then larger areas
 * first; equal areas in label order).  targets (room for n_labels rows) gets the rows in that order, plane[pos] the
 * label row, counts (n_images + 1) = [total, kept per image]. */
int y5_seg_order(const int32_t* image_rows, int32_t n_images, const int32_t* keep, const int32_t* areas, const float* rows,
                 int32_t overlap, float* targets, int32_t* plane, int32_t* counts, void* stream);
/* The batch's masks: overlap -> n_out = n_images planes, v = clip(v + m_i * (i + 1), 0, i + 1) over the image's labels in
 * order, in uint8 (with its wrap-around) up to 255 labels, else int32; otherwise n_out = total planes, one per label.
 * Flips from the table; out_dtype Y5_U8 | Y5_SEG_I32 | Y5_F32. */
int y5_seg_compose(const y5_aug_image* table, const y5_aug_label* labels, const int32_t* counts, const int32_t* plane,
                   const uint8_t* masks, int32_t n_out, int32_t mask_h, int32_t mask_w, int32_t overlap, void* out, int32_t out_dtype,
                   void* stream);

/* Classification head (models/common.py:1120-1140 Classify) and loss (utils/torch_utils.py:52-57 smartCrossEntropyLoss).
 * Global average pool over an NHWC channel-slice view x (B, h, w, pitch x_pitch): y[b * y_pitch + c] = the h*w pixels of
 * channel c summed in fp32 in pixel order, divided by h*w and rounded once to the dtype (Y5_F16 | Y5_BF16; c, pitches % 8).
 * No atomics: the result repeats bit for bit. */
int y5_global_avg_pool(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                       int32_t dtype, void* stream);
/* Its backward: dx (B, h, w, pitch dx_pitch) = dy[b * dy_pitch + c] / (h*w) at every pixel, computed in fp32, rounded once. */
int y5_global_avg_pool_bwd(const void* dy, int32_t dy_pitch, void* dx, int32_t dx_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                           int32_t dtype, void* stream);
/* nn.CrossEntropyLoss(label_smoothing=eps) with reduction 'mean' on logits (batch, nc) with row stride `row_stride` elements
 * (Y5_F16 | Y5_BF16 | Y5_F32) and int64 labels (DEVICE):
 *   row_loss[b] = (1 - eps) * (lse - x[y]) + (eps / nc) * sum_c (lse - x[c]),  lse = max + log(sum exp(x - max)), in fp32;
 *   *loss       = sum_b row_loss[b] / batch, summed by one block in a fixed order (bitwise repeatable).
 * dlogits != NULL also writes, in the logits dtype with row stride dlogits_stride,
 *   dlogits[b][c] = g * (softmax[b][c] - q[b][c]) / batch,  q = (1 - eps) * onehot(y) + eps / nc,
 * g = *grad_scale (DEVICE fp32, the upstream gradient, e.g. GradScaler's factor; NULL: 1) multiplied in fp32 before the one
 * rounding.  A label outside [0, nc) gives a NaN row loss (so a NaN *loss) and NaN gradients for its row -- there is no device
 * assert and no ignore_index.  row_loss: DEVICE scratch of `batch` floats.  No host synchronisation; nc >= 2, any size. */
int y5_cross_entropy(const void* logits, int32_t dtype, int32_t batch, int32_t nc, int64_t row_stride, const int64_t* labels,
                     float label_smoothing, const float* grad_scale, void* dlogits, int64_t dlogits_stride, float* row_loss, float* loss,
                     void* stream);

/* Validation AP (utils/metrics.py:25-126 ap_per_class, utils/segment/metrics.py:17-64 ap_per_class_box_and_mask) in float64.
 * Rows: image b (0 <= b < n_img) holds rows r < count[b] (clamped to [0, rows_per_image]; count NULL: all), read in (image, row)
 * order -- the flat form is n_img = 1, count NULL.  Row (b, r): conf / pred_cls at element b * img_stride + r * row_stride,
 * its niou tp values (uint8, nonzero = true) at tp + b * tp_img_stride + r * tp_row_stride; tp2 (NULL or the same layout)
 * is a second tp matrix evaluated on the same order (box and mask).  target_cls: nt labels.  Class values must be integers in
 * [0, 4096); any other value sets a flag in meta[2] (1: a prediction, 2: a label) and its row counts as class 0.
 * Order: np.argsort(-conf, kind="stable") (equal confidences keep row order, NaN last).  grid (DEVICE, 1101 float64):
 * np.linspace(0, 1, 1000) then np.linspace(0, 1, 101).  nc_cap = min(nt, 4096).  Outputs (DEVICE):
 *   out : per set s, at out + s * nc_cap * (5 + niou): tp, fp, p, r, f1 (nc_cap float64 each, at the max mean-F1 index),
 *         then ap (nc_cap x niou); the first nc entries (rows) are valid
 *   meta: Y5_AP_META + nc_cap int32 = [rows, nc, flags, max-F1 index of set 0, of set 1, unique classes ascending (nc)]
 * Every output but the max-F1 index equals the reference's float64 bits at that index; the index comes from the smoothed
 * mean-F1 curve, whose np.convolve summation order is not reproduced.  niou 1..32 (Y5_E_UNSUPPORTED above),
 * n_img * rows_per_image < 2^31.  No allocation and no host synchronisation; workspace: y5_ap_workspace_bytes, sets = 1 or 2. */
#define Y5_AP_META 5
int64_t y5_ap_workspace_bytes(int32_t n_img, int32_t rows_per_image, int32_t niou, int32_t nt, int32_t sets);
int y5_ap_per_class(const uint8_t* tp, const uint8_t* tp2, int64_t tp_img_stride, int32_t tp_row_stride, const float* conf,
                    const float* pred_cls, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t n_img,
                    int32_t rows_per_image, int32_t niou, const float* target_cls, int32_t nt, const double* grid, double eps,
                    void* workspace, int64_t workspace_bytes, double* out, int32_t* meta, void* stream);

/* Fused multi-head softmax attention (nn.MultiheadAttention's core with dropout 0, as the C3TR transformer layers run it):
 * per image b and head h, O = softmax(scale * Q K^T) V over `seq` tokens.  Token l of image b is row b*seq + l of each view;
 * head h owns the channels [h*head_dim, (h+1)*head_dim) of q, k, v (rows of `qkv_pitch` elements, e.g. the Q | K | V channel
 * slices of one (batch*seq, 3c) buffer) and of o (rows of `o_pitch`).  Other channels are neither read nor written.
 * head_dim 32, 64, 96, 128 or 160 (Y5_E_UNSUPPORTED otherwise); dtype Y5_F16 | Y5_BF16; any seq >= 1.  q, k, v, o 16-byte
 * aligned, pitches multiples of 8 and >= heads*head_dim (Y5_E_INVALID otherwise).  Products in fp32, online softmax in fp32,
 * O rounded once.  lse (optional, 4-byte aligned): the natural logsumexp of every row's scaled logits, [batch][heads][seq]
 * fp32, which y5_attention_bwd needs.  No L x L tensor is written; no allocation, no synchronisation. */
int y5_attention_fwd(const void* q, const void* k, const void* v, int32_t qkv_pitch, void* o, int32_t o_pitch, float* lse, int32_t batch,
                     int32_t seq, int32_t heads, int32_t head_dim, float scale, int32_t dtype, void* stream);
/* Its backward: dq, dk, dv (rows of `dqkv_pitch`, head channels as above) from q, k, v, o, dout (rows of `dout_pitch`) and the
 * forward's lse.  P is recomputed tile by tile from lse; delta is a workspace of batch*heads*seq fp32 (the row sums of
 * dout * o).  Same argument rules as y5_attention_fwd; every pointer is required.  Three launches, no atomics: the result
 * repeats bit for bit. */
int y5_attention_bwd(const void* q, const void* k, const void* v, int32_t qkv_pitch, const void* o, int32_t o_pitch, const void* dout,
                     int32_t dout_pitch, const float* lse, float* delta, void* dq, void* dk, void* dv, int32_t dqkv_pitch, int32_t batch,
                     int32_t seq, int32_t heads, int32_t head_dim, float scale, int32_t dtype, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Depthwise 5x5 / stride 1 / pad 2 conv of GhostConv's cheap half (models/common.py GhostConv.cv2 = Conv(c_, c_, 5, 1, None, c_))
 * over NHWC views of c channels (h x w), dtype Y5_F16 | Y5_BF16.
 *   weight : [c][5][5] in the activation dtype (the (c, 1, 5, 5) filter, y5_fold_pack with in_c = in_c_pad = 1), BN folded in
 *   bias   : fp32 [c] or NULL
 * y5_dwconv_fwd: y = act(fp32(sum of the 25 taps) + bias) + residual, the activation and residual as in y5_conv_desc, rounded
 * once.  flip != 0 rotates the taps 180 degrees: with bias NULL and Y5_ACT_NONE that is the data gradient dx of the conv from
 * dy = x, and `residual` adds another gradient of x in the same pass.  x_out (optional) receives x + x_res (x_res optional) at
 * every pixel: GhostBottleneck's first concat half, or a copy of x.  y may alias residual and x_out may alias x_res (in-place
 * adds); x may alias no output.  residual, x_res, x_out: NULL or views like x.
 * y5_dwconv_wgrad: fp32 dweight [c][5][5] = sum over (n, y, x) of x[n, y+ky-2, x+kx-2, c] * dy[n, y, x, c] (dweight is
 * overwritten).  The partial sums are added with fp32 atomics, so the last bits depend on scheduling (as y5_conv_wgrad).
 * Y5_E_INVALID for: ksize != 5 or stride != 1, c not a positive multiple of 8, a pitch < c or not a multiple of 8, a view not
 * 16-byte aligned, weight / bias / dweight not 4-byte aligned. */
int y5_dwconv_fwd(const void* x, int32_t x_pitch, const void* weight, const float* bias, void* y, int32_t y_pitch, const void* residual,
                  int32_t res_pitch, const void* x_res, int32_t x_res_pitch, void* x_out, int32_t x_out_pitch, int32_t batch, int32_t h,
                  int32_t w, int32_t c, int32_t ksize, int32_t stride, int32_t act, float act_slope, int32_t flip, int32_t dtype,
                  void* stream);
int y5_dwconv_wgrad(const void* x, int32_t x_pitch, const void* dy, int32_t dy_pitch, float* dweight, int32_t batch, int32_t h, int32_t w,
                    int32_t c, int32_t ksize, int32_t stride, int32_t dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* Y5B200_H */
