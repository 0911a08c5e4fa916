/*
 * yolort_b200 -- C ABI of the H100-native (sm_90a) YOLOv5 inference path.
 *
 * The reference (zhiqwang/yolort) has no FFI on this path: its boundary is the Python nn.Module
 * surface (yolort/models/yolov5.py:135 YOLOv5.forward, yolort/models/yolo.py:141 YOLO.forward).
 * These entry points sit directly under the Python classes of `yolort_b200.models` that mirror that
 * surface; each one states which reference function it replaces.
 *
 * Conventions: plain C, no torch types.  Every pointer named `*_dev` (and every tensor pointer
 * inside the structs) is a DEVICE pointer owned by the caller; `stream` is a `cudaStream_t` passed
 * as `void*`.  Functions return YB_OK (0) or a negative status; `yb_last_error()` gives the text of
 * the last failure on the calling thread.  Nothing is allocated or freed across the ABI except the
 * opaque plan handle.  There is no CPU fallback anywhere behind this ABI.
 */
#ifndef YOLORT_B200_H
#define YOLORT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YB_OK 0
#define YB_ERR_INVALID (-1)   /* bad argument / unsupported configuration */
#define YB_ERR_CUDA (-2)      /* CUDA runtime / driver error             */
#define YB_ERR_WORKSPACE (-3) /* workspace too small                     */

/* element types */
#define YB_U8 0
#define YB_F16 1
#define YB_BF16 2
#define YB_F32 3

const char* yb_last_error(void);
int yb_abi_version(void);

/* ------------------------------------------------------------------------------------------------
 * Letterbox  (replaces YOLOTransform.forward: yolort/models/transform.py:143-221, i.e.
 * _resize_image_and_masks :53-97 + batch_images :297-330)
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t src_h, src_w;     /* original image size                                         */
  int32_t new_h, new_w;     /* size after the aspect-preserving resize: int(in * scale)   */
  int32_t top, left;        /* paste offset inside the batch canvas                        */
  float ratio_h, ratio_w;   /* recomputed sampling ratios src/new (recompute_scale_factor) */
} yb_letterbox_geom;

/* Host-only geometry (no GPU needed): transform.py:66-73 scale rule (fp32 reciprocal-multiply),
 * F.interpolate output size int(in*scale), batch shape ceil-to-stride (:307-314) or fixed_shape,
 * centred offsets int(round(d/2 - 0.1)) (:322-326).  batch_hw receives {Hb, Wb}. */
int yb_letterbox_geometry(int n, const int32_t* src_hw, float min_size, float max_size,
                          int size_divisible, const int32_t* fixed_shape_or_null,
                          yb_letterbox_geom* geom_out, int32_t* batch_hw);

/* destination layouts */
#define YB_LAYOUT_NCHW 0  /* reference layout [N,3,Hb,Wb]                                          */
#define YB_LAYOUT_S2D16 1 /* [N,Hb/2,Wb/2,16]: channel (dy*2+dx)*4+c, c==3 is zero; feeds the stem */

/* Bilinear resize (align_corners=False, no antialias) + pad with `fill` + dtype/layout conversion
 * for the whole batch in one launch.  `src_dev[i]` is a device pointer to image i in CHW order
 * (row stride = src_w); uint8 sources are mapped through u8_lut_dev[256] (the caller decides how
 * u8 maps to [0,1]; the Python layer fills it with torch's `u8 / 255.0`). */
int yb_letterbox(int n, const void* const* src_dev, int src_dtype, const yb_letterbox_geom* geom,
                 int Hb, int Wb, float fill, const float* u8_lut_dev, void* dst_dev, int dst_dtype,
                 int dst_layout, void* stream);

/* Same, with an explicit source memory order: YB_SRC_CHW (planar, what yb_letterbox assumes) or YB_SRC_HWC
 * (interleaved RGBRGB..., what image decoders emit -- the output of the reference's default loader
 * `read_image` (yolort/models/yolov5.py:218-228) before its permute), so decoded files go from a pinned
 * host buffer to the canvas without a repacking pass. */
#define YB_SRC_CHW 0
#define YB_SRC_HWC 1
int yb_letterbox_strided(int n, const void* const* src_dev, int src_dtype, int src_layout,
                         const yb_letterbox_geom* geom, int Hb, int Wb, float fill, const float* u8_lut_dev,
                         void* dst_dev, int dst_dtype, int dst_layout, void* stream);

/* Host-only: scale_coords parameters of transform.py:354-367 for one image:
 * out[0]=gain, out[1]=pad_x, out[2]=pad_y (all fp32, fractional pads). */
int yb_scale_coords_params(int Hb, int Wb, int src_h, int src_w, float* out3);

/* ------------------------------------------------------------------------------------------------
 * Convolution plan  (replaces BackboneWithPAN.forward + YOLOHead.forward:
 * yolort/models/backbone_utils.py:54-57, path_aggregation_network.py:199-239, box_head.py:68-82;
 * blocks from yolort/v5/models/common.py:42-207)
 * ---------------------------------------------------------------------------------------------- */
#define YB_OP_CONV 0       /* act(conv(x) * bn_scale + bn_shift) [+ residual]; BN pre-folded      */
#define YB_OP_SPP_POOL 1   /* y[c:2c]=mp5(x) y[2c:3c]=mp9(x) y[3c:4c]=mp13(x), stride 1, -inf pad */
#define YB_OP_UPSAMPLE2X 2 /* nearest x2 (nn.Upsample(scale_factor=2))                            */

#define YB_ACT_NONE 0
#define YB_ACT_SILU 1
#define YB_ACT_HARDSWISH 2 /* r3.1 Conv (yolort/v5/models/common.py:64)              */
#define YB_ACT_LEAKY01 3   /* r3.1 BottleneckCSP: LeakyReLU(0.1) after the concat BN (:141-142) */

/* Optional fused post-processing of a detection-head convolution (yolort/models/box_head.py:68-82 followed by
 * :328-360,418): instead of storing the logits, the epilogue applies sigmoid / anchor decode / multi-label
 * threshold to the fp32 accumulators and appends candidates straight into the NMS workspace (see
 * yb_nms_layout).  The head must fit one N tile (n_anchors * (n_classes + 5) <= 256). */
typedef struct {
  int32_t n_anchors, n_classes;
  int32_t level_start;        /* flat index of this level's first anchor inside an image     */
  int32_t anchors_per_image;  /* over all levels                                             */
  float stride_px;
  float anchors_px[8];        /* (w, h) per anchor, pixels                                   */
  float score_thresh;
  int64_t cap_per_image;      /* candidate slots per image in `keys`                         */
  uint64_t* keys;             /* [n][cap_per_image]                                          */
  void* boxes;                /* float4 [n][anchors_per_image]                               */
  int32_t* img_count;         /* [n]                                                         */
  int32_t* img_maxc;          /* [n] ordered-int max box coordinate                          */
} yb_head_decode;

/* Optional pointwise tail chained onto a convolution INSIDE the same kernel: the 1x1 convolution that consumes the
 * first convolution's output tile straight from shared memory (the epilogue's swizzled staging box is exactly the
 * K-major operand tile the tensor core reads), so the intermediate never makes an HBM round trip and one launch
 * boundary disappears.  Covers the pointwise chains of the reference's C3 / Bottleneck blocks
 * (yolort/v5/models/common.py:94-116,149-173):
 *   cv1||cv2 -> m.0.cv1          (own_C = c of the 2c output channels feed the tail; the first output is stored)
 *   m.i.cv2 (3x3 + shortcut) -> m.(i+1).cv1
 *   m.last.cv2 (3x3 + shortcut) -> cv3 over cat(m_out, cv2(x)): `extra` is the cv2 half, first output not stored
 * tail(x) = act(W2 . [first_out[0:own_C] | extra] + bias2).  Supported when yb_conv_chain_supported() says so. */
typedef struct {
  const void* weight;           /* [Cout_pad][K_pad] K-major, K = own_C + extra_C (own channels first)          */
  const float* bias;            /* [Cout_pad] fp32                                                                */
  int32_t Cout, Cout_pad, K_pad;
  int32_t act;
  void* out;                    /* NHWC view at the first convolution's OUTPUT resolution                         */
  int32_t out_cstride;
  int32_t own_C;                /* channels [0, own_C) of the first convolution's output feed the tail           */
  const void* extra;            /* optional second operand block (NHWC view, output resolution), may be NULL      */
  int32_t extra_C, extra_cstride;
  int32_t store_first;          /* 0: the first convolution's output stays on chip (nothing is written to `out`
                                   of the op itself); 1: it is stored as usual                                    */
} yb_conv_chain;

/* All activation tensors are NHWC views: element (n,y,x,c) at base[((n*H+y)*W+x)*cstride + c].
 * `cstride` >= channels lets a producer write straight into a slice of a concat buffer. */
typedef struct {
  int32_t kind;
  int32_t dtype;                /* YB_F16 or YB_BF16 (accumulation is always fp32) */
  int32_t N, H, W;              /* input spatial extent                              */
  int32_t Cin, in_cstride;
  const void* in;
  int32_t Ho, Wo;               /* output spatial extent                             */
  int32_t Cout, out_cstride;
  void* out;
  int32_t ksize, stride, pad;
  int32_t act;
  const void* weight;           /* [Cout_pad][ksize*ksize][Cin_pad], K contiguous, zero padded   */
  int32_t Cin_pad, Cout_pad;
  const float* bias;            /* [Cout_pad] fp32 (folded BN shift, or the head's conv bias)     */
  const void* residual;         /* optional NHWC view added after the activation (Bottleneck)    */
  int32_t res_cstride;
  int32_t reserved;             /* bit 0: keep a 3x3 conv on the generic im2col kernel; bit 1: `weight` is the banded
                                   super-pixel stem matrix [Cout_pad][3][128] (engine.stem_band); bit 2: take the
                                   halo-patch kernel's stride-2 parity-plane variant whatever the channel counts (tests);
                                   bit 3: do not split N over CTAs with resident weights (A/B timing, tests);
                                   other bits: must be zero */
  const yb_head_decode* decode; /* optional (host pointer, copied at plan creation): fused decode epilogue */
  const yb_conv_chain* chain;   /* optional (host pointer, copied at plan creation): chained pointwise tail  */
} yb_op_desc;

/* 1 if `op` (a YB_OP_CONV with op->chain set) can run as one fused launch on this build, else 0 (the caller then
 * emits the two convolutions separately).  Pure host logic: no GPU needed. */
int yb_conv_chain_supported(const yb_op_desc* op);

/* Host-only introspection of how a convolution would be launched (tests, tuning): fills 12 ints
 *   [0] 1 = halo-patch kernel, 0 = im2col / 1x1 kernel   [1] N-tile width   [2] N tiles   [3] weights resident in
 *   shared memory   [4] M tiles per weight pass   [5] patch slots (pipeline stages)   [6] weight-ring slabs (k-iterations
 *   per stage)   [7] store-box columns   [8] staging buffers per epilogue group (halo-patch kernel) / epilogue groups
 *   (1x1 / im2col kernel)   [9] dynamic shared memory   [10] grid
 *   [11] chained tail fused.  Pure host logic. */
int yb_conv_config(const yb_op_desc* op, int32_t* info12);

typedef struct yb_plan yb_plan;

/* Validates every op, builds the TMA descriptors and launch configurations once. */
int yb_plan_create(const yb_op_desc* ops, int n_ops, yb_plan** plan_out);
/* Enqueues every kernel of the plan on `stream` (graph-capturable: no host sync, no allocation). */
int yb_plan_run(yb_plan* plan, void* stream);
/* Runs ops [first, first+count) only (profiling / stage-wise parity). */
int yb_plan_run_range(yb_plan* plan, int first, int count, void* stream);
int yb_plan_num_launches(const yb_plan* plan);
int yb_plan_destroy(yb_plan* plan);

/* ------------------------------------------------------------------------------------------------
 * Post-process  (replaces PostProcess.forward: yolort/models/box_head.py:388-429 incl.
 * _concat_pred_logits :328-348, det_utils.decode_single _utils.py:43-62, _decode_pred_logits
 * :351-360, torchvision.ops.batched_nms, and YOLOTransform.postprocess transform.py:332-367)
 * ---------------------------------------------------------------------------------------------- */
#define YB_MAX_LEVELS 4
#define YB_MAX_ANCHORS 4

typedef struct {
  const void* logits;   /* raw head outputs (pre-sigmoid)                                        */
  int32_t dtype;        /* YB_F16 / YB_BF16 / YB_F32                                             */
  int32_t H, W;
  /* element strides of logit (n, a, y, x, k); k (0..nc+4) is contiguous */
  int64_t stride_n, stride_a, stride_y, stride_x;
  float stride_px;                       /* level stride in pixels (8/16/32)  */
  float anchors_px[2 * YB_MAX_ANCHORS];  /* (w,h) per anchor in pixels        */
} yb_head_level;

#define YB_NMS_TV_AUTO 0         /* branch like torchvision CPU: offset trick iff 4*cands <= 4000 */
#define YB_NMS_EXACT_PER_CLASS 1 /* suppress only within a class, exact coordinates                */
#define YB_NMS_OFFSET_TRICK 2    /* boxes + label*(max_coord+1) in fp32, class-agnostic sweep      */

typedef struct {
  int32_t n_images, n_levels, n_anchors, n_classes;
  float score_thresh, iou_thresh;
  int32_t max_det;       /* detections_per_img (<= 4096)                                          */
  int32_t semantics;
  int64_t max_candidates; /* capacity of the candidate arena for the whole batch                  */
} yb_nms_params;

size_t yb_decode_nms_workspace_bytes(const yb_nms_params* p, const yb_head_level* levels);
/* Debug aid: byte offset inside the workspace of 16 int64 words; words [4,10) hold the clock counts of the
 * NMS kernel's phases for image 0 of the last call (sort, kept-list test, compaction, bit-matrix, resolve, rest). */
size_t yb_decode_nms_debug_offset(const yb_nms_params* p, const yb_head_level* levels);

/* Outputs are padded to max_det per image: boxes [n][max_det][4] fp32 (xyxy, rescaled to the
 * original image if rescale_dev != NULL: [n][3] = gain, pad_x, pad_y), scores [n][max_det],
 * labels [n][max_det] int64, counts [n] int32.  status_dev is int64[4]: [0] = total number of
 * candidates found, [1] = 1 if some image exceeded its share max_candidates/n_images of the arena
 * (its result is then empty: grow and re-run), [2] = largest per-image candidate count. */
int yb_decode_nms(const yb_nms_params* p, const yb_head_level* levels, const float* rescale_dev,
                  float* boxes_dev, float* scores_dev, int64_t* labels_dev, int32_t* counts_dev,
                  int64_t* status_dev, void* workspace_dev, size_t workspace_bytes, void* stream);

/* The same pipeline in pieces, for plans whose head convolutions carry the fused decode epilogue:
 * yb_nms_layout reports where inside `workspace_dev` the candidate arena lives (what yb_head_decode needs),
 * yb_nms_begin zeroes the per-image counters, [the plan runs], yb_nms_finish sorts + suppresses + writes. */
typedef struct {
  uint64_t* keys;
  void* boxes;
  int32_t* img_count;
  int32_t* img_maxc;
  int64_t cap_per_image;
  int32_t anchors_per_image;
  int32_t level_start[YB_MAX_LEVELS];
} yb_nms_layout_t;
int yb_nms_layout(const yb_nms_params* p, const yb_head_level* levels, void* workspace_dev, size_t workspace_bytes,
                  yb_nms_layout_t* out);
int yb_nms_begin(const yb_nms_params* p, const yb_head_level* levels, int64_t* status_dev, void* workspace_dev,
                 size_t workspace_bytes, void* stream);
int yb_nms_finish(const yb_nms_params* p, const yb_head_level* levels, const float* rescale_dev, float* boxes_dev,
                  float* scores_dev, int64_t* labels_dev, int32_t* counts_dev, int64_t* status_dev,
                  void* workspace_dev, size_t workspace_bytes, void* stream);
/* The decode + multi-label threshold step alone (box_head.py:328-360, :418): appends the candidates of `levels` to the
 * workspace arena between yb_nms_begin and yb_nms_finish.  yb_decode_nms == begin + decode_candidates + finish; the
 * split exists so that a caller can time (or overlap) the three steps separately. */
int yb_decode_candidates(const yb_nms_params* p, const yb_head_level* levels, void* workspace_dev,
                         size_t workspace_bytes, void* stream);

/* Dense decode, no threshold / NMS (replaces LogitsDecoder.forward: yolort/relay/logits_decoder.py:26-61, the
 * output the reference hands to TensorRT's EfficientNMS plugin): boxes_dev [n_images, anchors_per_image, 4] fp32
 * xyxy and scores_dev [n_images, anchors_per_image, n_classes] fp32 = sigmoid(cls) * sigmoid(obj), anchors in the
 * reference's concatenation order (level, anchor, y, x). Only n_images/n_levels/n_anchors/n_classes of `p` are read. */
int yb_decode_dense(const yb_nms_params* p, const yb_head_level* levels, float* boxes_dev, float* scores_dev,
                    void* stream);

/* torchvision.ops.batched_nms on explicit candidates (one image), first `max_keep` survivors in
 * score-descending order (ties: lower index first).  keep_dev [max_keep] int64, n_keep_dev [1]. */
size_t yb_batched_nms_workspace_bytes(int64_t n_boxes);
int yb_batched_nms(const float* boxes_dev, const float* scores_dev, const int64_t* labels_dev,
                   int64_t n_boxes, float iou_thresh, int semantics, int32_t max_keep,
                   int64_t* keep_dev, int32_t* n_keep_dev, void* workspace_dev,
                   size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YOLORT_B200_H */
