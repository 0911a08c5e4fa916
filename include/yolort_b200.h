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
#define YB_F8E4M3 4 /* float8 e4m3 ("fn": max 448, no infinities); values are stored divided by a power-of-two scale */

const char* yb_last_error(void);
/* 2 since yb_conv_config fills a yb_conv_info; it filled twelve ints at 1 */
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

/* One test-time-augmentation canvas (scale_img, yolort/v5/utils/torch_utils.py:288-300, of the canvas or of its
 * left-right mirror): n space-to-depth canvases [n, Hb/2, Wb/2, 16] (fp16 or bf16) -> [n, Hp/2, Wp/2, 16] of the same
 * dtype.  Pixels [0, nh) x [0, nw) are the bilinear resize (align_corners=False, ratios float(Hb)/nh, float(Wb)/nw,
 * fp32 arithmetic, one rounding) of the canvas, mirrored when flip_lr; the rest is `fill`; channel 3 is zero. */
int yb_canvas_rescale(int n, const void* src_dev, int dtype, int Hb, int Wb, int nh, int nw, int flip_lr, float fill,
                      void* dst_dev, int Hp, int Wp, void* stream);

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
#define YB_OP_ATTENTION 3  /* multi-head softmax(Q_h K_h^T / sqrt(d)) V_h over the H*W tokens of each image  */
#define YB_OP_DWCONV 4     /* depthwise k x k convolution, one group per channel (MobileNetV3 InvertedResidual)  */
#define YB_OP_SE 5         /* in-place squeeze-excitation x <- x * hardsigmoid(W2 relu(W1 mean_hw(x) + b1) + b2)  */
#define YB_OP_AVGPOOL 6    /* global average pool y[n,0,0,c] = mean_hw(x[n,:,:,c]) (nn.AdaptiveAvgPool2d(1))       */
#define YB_OP_QUANTIZE 7   /* y = RN_satfinite(x / s) to e4m3, one power-of-two scale s per tensor (FP8 plans)      */

#define YB_ACT_NONE 0
#define YB_ACT_SILU 1
#define YB_ACT_HARDSWISH 2 /* r3.1 Conv (yolort/v5/models/common.py:64)              */
#define YB_ACT_LEAKY01 3   /* r3.1 BottleneckCSP: LeakyReLU(0.1) after the concat BN (:141-142) */
#define YB_ACT_RELU 4      /* MobileNetV3 "RE" blocks (torchvision mobilenetv3.py)              */

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
/* YB_OP_ATTENTION (the nn.MultiheadAttention core of the reference's TransformerLayer, yolort/v5/models/common.py:
 * 308-331; its in- and out-projections are YB_OP_CONV 1x1 ops) reads the fields as follows:
 *   in:        the packed [q | k | v] NHWC view, Cin = 3E, in_cstride >= 3E
 *   out:       an NHWC view, Cout = E, out_cstride >= E
 *   N, H, W:   the sequence of image n is its L = H*W pixels in row-major order; Ho == H, Wo == W
 *   ksize:     the number of heads; head h reads channels [h*d, (h+1)*d) of each third and writes the same window
 *              of `out`, d = E / heads = 64 (the only head width implemented)
 *   weight, bias, residual, decode and chain must be NULL; act and reserved must be 0; Cin_pad, Cout_pad, stride,
 *   pad and res_cstride are not read.
 * The op computes softmax(Q_h K_h^T / sqrt(d)) V_h for every image and head, with no mask, fp32 softmax and
 * accumulation.  Channel counts and strides must be multiples of 8 and both tensors 16-byte aligned. */
/* YB_OP_DWCONV (the depthwise convolution of torchvision's InvertedResidual, yolort/models/yolo_lite.py:74-105; also
 * the stride-2 subsample of the FPN's LastLevelMaxPool, as ksize 1 with unit weights) reads the fields as follows:
 *   in, out:   NHWC views with Cin == Cout == C, C and both cstrides multiples of 8
 *   ksize, stride, pad:  ksize in {1, 3, 5}, stride in {1, 2}, pad == ksize / 2, zero padding;
 *              Ho == (H + 2 pad - ksize) / stride + 1, Wo likewise
 *   act:       YB_ACT_NONE, YB_ACT_RELU or YB_ACT_HARDSWISH
 *   weight:    [ksize * ksize][C] in the compute dtype (tap-major, channels contiguous; BN folded)
 *   bias:      [C] fp32
 *   residual, decode and chain must be NULL, reserved 0; Cin_pad, Cout_pad and res_cstride are not read.
 * out[n,y,x,c] = act(sum_ij w[i*k+j][c] * in[n, y*s-p+i, x*s-p+j, c] + b[c]), fp32 accumulation, one rounding.
 * in, out and weight must be 16-byte aligned, bias 4-byte aligned.
 *
 * YB_OP_SE (torchvision.ops.SqueezeExcitation inside InvertedResidual) works in place and reads the fields as follows:
 *   in, out:   the same NHWC view (in == out, in_cstride == out_cstride), Cin == Cout == C, C <= 2048 a multiple of 8;
 *              Ho == H, Wo == W
 *   ksize:     the squeeze width S (fc1: C -> S, fc2: S -> C), 1 <= S <= 1024
 *   weight:    fp32 [C][S] (W1 transposed: fc1.weight[s][c] at [c*S + s]) followed by fp32 [S][C] (W2 transposed:
 *              fc2.weight[c][s] at [C*S + s*C + c])
 *   bias:      fp32 [S] (fc1.bias) followed by fp32 [C] (fc2.bias)
 *   act, stride and pad are not read; residual, decode and chain must be NULL, reserved 0.
 * Per image: m = mean_hw(x) in fp32, g = hardsigmoid(W2 relu(W1 m + b1) + b2), x <- round(x * g).  The mean is summed
 * in a fixed order without atomics (a repeated run gives the same bits).  weight and bias must be 16-byte aligned.
 *
 * YB_OP_AVGPOOL (the AdaptiveAvgPool2d(1) of the DarkNet classifiers, yolort/models/darknetv4.py, darknetv6.py) reads
 * the fields as follows:
 *   in, out:   NHWC views with Cin == Cout == C, C and both cstrides multiples of 8; N <= 65535
 *   Ho, Wo:    1 (the output view holds one pixel per image: out[n*out_cstride + c])
 *   weight, bias, residual, decode and chain must be NULL; act and reserved must be 0; ksize, stride, pad, Cin_pad,
 *   Cout_pad and res_cstride are not read.
 * out[n,0,0,c] = round(sum_{y,x} in[n,y,x,c] / (H*W)): the sum is fp32 in a fixed order without atomics (a repeated
 * run gives the same bits), divided once and rounded once to the compute dtype.  in and out must be 16-byte aligned.
 *
 * FP8 (e4m3) plans.  An e4m3 tensor stores x / s for one power-of-two scale s per tensor (per output channel for conv
 * weights); every conversion to e4m3 rounds to nearest even and saturates at +-448 (cvt.rn.satfinite: never a NaN).
 * Channel counts, channel offsets and cstrides of e4m3 views are multiples of 16 (16 bytes), like every 16-byte view.
 * YB_OP_CONV with dtype YB_F8E4M3 (the FP8 implicit-GEMM kernel) reads the fields as follows:
 *   in, residual:  e4m3 NHWC views (scales s_in, s_res); Cin, in_cstride and res_cstride multiples of 16
 *   out:       an e4m3 NHWC view (scale s_out), Cout and out_cstride multiples of 16; or, with YB_CONV_E4M3_F16_OUT
 *              (YB_CONV_E4M3_BF16_OUT), an fp16 (bf16) NHWC view, Cout and out_cstride multiples of 8, that gets the
 *              dequantised values (head logits)
 *   ksize, stride, pad:  1x1/s1/p0, 3x3/s1/p1 or 3x3/s2/p1
 *   act:       YB_ACT_NONE, SILU, HARDSWISH, LEAKY01 or RELU
 *   weight:    e4m3 [Cout_pad][ksize*ksize][Cin_pad], Cin_pad a multiple of 32 (the K step), zero padded; row c holds
 *              w[c] / s_w[c]
 *   bias:      fp32 [Cout_pad] bias, then fp32 [Cout_pad] multipliers m[c] = s_w[c] * s_in, then {s_res, 1/s_out}
 *   reserved:  YB_CONV_E4M3_F16_OUT or YB_CONV_E4M3_BF16_OUT, every other bit zero; decode and chain must be NULL;
 *              a residual needs the e4m3 output.
 *   v = act(acc * m[c] + bias[c]) [+ res * s_res] with the e4m3 dot product acc accumulated in fp32, then
 *   out = RN_satfinite(v * (1/s_out)) (e4m3) or RN(v) (fp16 / bf16).
 * YB_OP_QUANTIZE: dtype is the SOURCE type (YB_F16 or YB_BF16); in is that NHWC view, out an e4m3 NHWC view of the
 *   same extent (Ho == H, Wo == W, Cout == Cin, a multiple of 16; in_cstride a multiple of 8, out_cstride of 16);
 *   bias: fp32 {1/s}; weight, residual, decode and chain NULL; act and reserved 0.  out = RN_satfinite(in * (1/s)).
 * YB_OP_SPP_POOL and YB_OP_UPSAMPLE2X with dtype YB_F8E4M3: source and destination share one scale, so the pool is a
 *   max over the decoded values and the upsample a copy, both exact; channel counts and cstrides multiples of 16.
 * FP8 left yb_abi_version() unchanged: the descriptor layout is the same, and the element type, the op kind and the
 * reserved bits are additions that every earlier descriptor leaves at values it already had to use. */
typedef struct {
  int32_t kind;
  int32_t dtype;                /* YB_F16, YB_BF16 or YB_F8E4M3 (accumulation is always fp32) */
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
  int32_t reserved;             /* option bits of a convolution (YB_CONV_* below); other bits: must be zero */
  const yb_head_decode* decode; /* optional (host pointer, copied at plan creation): fused decode epilogue */
  const yb_conv_chain* chain;   /* optional (host pointer, copied at plan creation): chained pointwise tail  */
} yb_op_desc;

/* yb_op_desc.reserved option bits of an fp16 / bf16 YB_OP_CONV: */
#define YB_CONV_FORCE_IM2COL 1   /* keep a 3x3 conv on the generic im2col kernel */
#define YB_CONV_BAND_STEM 2      /* `weight` is the banded super-pixel stem matrix [Cout_pad][3][128] (engine.stem_band) */
#define YB_CONV_FORCE_PLANES 4   /* take the halo-patch kernel's stride-2 parity-plane variant whatever the channel
                                    counts (tests) */
#define YB_CONV_NO_NSPLIT 8      /* do not split N over CTAs with resident weights (A/B timing, tests) */
#define YB_CONV_ONE_CTA 16       /* keep one CTA per SM where the shape would take two (tests compare the two launches
                                    bit for bit) */
#define YB_CONV_NO_TAIL_SPLIT 64 /* 1x1 / im2col kernel: run the last round's tiles whole instead of splitting them over
                                    the idle CTAs, and single tiles instead of two-tile tasks (tests compare the
                                    launches bit for bit, A/B timing) */
#define YB_CONV_PAIR_N64 128     /* halo-patch kernel: keep streamed-weight pair tasks at 64 columns on two consumer
                                    warpgroups instead of 128 columns on four; either kernel: keep two-team launches on
                                    two consumer warpgroups; 1x1 / im2col kernel: keep streamed-weight launches on single
                                    tiles of two consumer warpgroups instead of two-tile tasks on four: every launch on
                                    four runs on two (tests compare the two launches bit for bit, A/B timing) */
#define YB_CONV_NO_TEAMS 256     /* halo-patch and 1x1 / im2col kernels: keep chained and banded-stem launches on two
                                    consumer warpgroups instead of two teams of two (tests compare the two launches bit
                                    for bit, A/B timing) */
/* ... and of an e4m3 YB_OP_CONV (see above), which takes these two only: */
#define YB_CONV_E4M3_F16_OUT 16  /* fp16 output */
#define YB_CONV_E4M3_BF16_OUT 32 /* bf16 output */

/* 1 if `op` (a YB_OP_CONV with op->chain set) can run as one fused launch on this build, else 0 (the caller then
 * emits the two convolutions separately).  Pure host logic: no GPU needed. */
int yb_conv_chain_supported(const yb_op_desc* op);

/* How a convolution is launched (yb_conv_config). */
#define YB_CONV_KERNEL_IM2COL 0   /* the 1x1 / im2col kernel (conv_sm90.cu) */
#define YB_CONV_KERNEL_PATCH 1    /* the 3x3 halo-patch kernel (conv3x3_patch_sm90.cu) */
#define YB_CONV_KERNEL_E4M3 2     /* the e4m3 kernel (conv_fp8_sm90.cu) */
#define YB_CONV_TILING_ROWS 0     /* tiles of consecutive output rows M (1x1 / im2col and e4m3 kernels) */
#define YB_CONV_TILING_CLASSIC 1  /* halo patch: 16 x 8 pixel tiles */
#define YB_CONV_TILING_WRAP 2     /* halo patch: 5 x 24 pixel tiles of maps at most 22 pixels wide */
#define YB_CONV_TILING_STRIDE2 3  /* halo patch: 16 x 8 output pixels over two column-parity planes of the input */
typedef struct {
  int32_t kernel;            /* YB_CONV_KERNEL_* */
  int32_t block_n;           /* N-tile width (the wgmma N) */
  int32_t n_tiles;           /* N tiles */
  int32_t weights_resident;  /* the weights of the CTA's N tile stay in shared memory */
  int32_t tiles_per_pass;    /* M tiles per weight pass (2 when pairs of tiles share each weight slab) */
  int32_t slots;             /* pipeline stages (two teams of the 1x1 / im2col kernel: per team; halo patch: patch slots) */
  int32_t ring;              /* k-iterations per stage (halo patch: weight-ring slabs, 0 with resident weights) */
  int32_t store_cols;        /* store-box columns */
  int32_t store_bufs;        /* staging buffers per epilogue group */
  int32_t groups;            /* consumer warpgroups per CTA: 2, 1 (1x1 / im2col kernel, 64-row tiles) or 4 (halo patch:
                                128-column pair tasks; either kernel: two teams of single-tile tasks) */
  int32_t resident_ctas;     /* CTAs resident per SM: 1 or 2 */
  int32_t chained;           /* a chained tail is fused */
  int32_t smem_bytes;        /* dynamic shared memory per CTA */
  int32_t grid;              /* CTAs of the persistent grid */
  int32_t tiling;            /* YB_CONV_TILING_* */
  int32_t m_tiles;           /* output tiles along M */
  int32_t work_items;        /* tiles (halo patch: tasks) the grid walks */
  int32_t tail_n;            /* wgmma N of the chained tail, 0 without one */
  int32_t tail_tiles;        /* 1x1 / im2col kernel: tiles of the last round that are split along N, 0 if none */
  int32_t tail_split;        /* ... into this many sub-tasks each (1, or 0 from the other kernels: none) */
} yb_conv_info;

/* Host-only introspection of how a convolution would be launched (tests, tuning).  A convolution takes two CTAs per SM
 * of two consumer warpgroups each when its kernel has a two-CTA instance for the N tile (1x1 / im2col: N <= 64 with no
 * tail or a tail of at most 64 columns; halo patch: N = 32 or 64, or 32 with a 64-column tail, single-tile tasks,
 * resident weights in one N tile, no banded stem), its plan fits half of the SM's shared memory and it has at least
 * 2 x SMs tiles; the grid is then up to 2 x SMs.  Otherwise a 1x1 / im2col convolution takes two CTAs per SM of ONE
 * consumer warpgroup each (64-row tiles) when its one-CTA plan has a 256-column N tile and no chained tail and it has at
 * least 3 x SMs 128-row tiles: it then runs as two 128-column N tiles whose weights stay resident (at most 80 KB per N
 * tile, one N tile per CTA), in half of the SM's shared memory, on a grid of 2 x SMs.  A 1x1 / im2col convolution
 * with 128-column N tiles, no chained tail or fused decode and a grid that is a multiple of its N tiles splits the
 * r tiles of a partial last round in two when 2 r <= grid (64-row halves with two consumer warpgroups, 64-column halves
 * with one), which the otherwise idle CTAs run (tail_tiles = r, tail_split = 2); a one-CTA plan whose 256-column N
 * tile streams its weights over 2-4 rounds takes 128-column N tiles when that split then applies.  Reserved bit
 * YB_CONV_NO_TAIL_SPLIT keeps the tiles whole (and 256 columns).  A halo-patch convolution with streamed weights (pair
 * tasks) whose Cout is a multiple of 128 runs its pairs with 128-column N tiles on one CTA of four consumer warpgroups
 * (groups = 4) when the grid is a multiple of the N tiles and its T tasks satisfy T >= SMs and T mod SMs = 0 or
 * > SMs / 2; reserved bit YB_CONV_PAIR_N64 keeps the 64-column pairs.  A halo-patch convolution with resident weights
 * in one N tile, single-tile classic-tiled tasks and either a chained tail after a 64-column N tile or the banded stem
 * runs on one CTA of two consumer teams of two warpgroups each (groups = 4, tiles_per_pass 1) when it has at least
 * 8 x SMs tasks and the two teams' staging buffers fit in shared memory; reserved bit YB_CONV_NO_TEAMS keeps two
 * consumer warpgroups, as does YB_CONV_PAIR_N64.  A 1x1 / s1 convolution of one CTA per SM with a 128-column N tile of
 * resident weights over whole 64-channel K chunks, chained to a 64-column tail over one or two 64-channel boxes, runs
 * on two consumer teams too (groups = 4, layout 1x4, one k-iteration per stage and `slots` stages per team) when it
 * has at least 8 x SMs tiles and the weights, both teams' staging buffers and two stages per team fit in shared
 * memory; reserved bits YB_CONV_NO_TEAMS, YB_CONV_PAIR_N64 and YB_CONV_ONE_CTA keep two consumer warpgroups.  A
 * one-CTA 1x1 / im2col convolution that streams its weights in 128-column N tiles over whole 64-channel K chunks,
 * without a residual, chained tail or fused decode, runs as tasks of two 128-row M tiles sharing each weight slab on
 * four consumer warpgroups (groups = 4, tiles_per_pass 2, layout 1x4x2 in _C.conv_config) when it has at least 100 M
 * tiles and either at most one per SM, three or more N tiles or at least 400 M tiles, and the grid min(tasks, SMs) is
 * a multiple of the N tiles; reserved bits YB_CONV_PAIR_N64, YB_CONV_ONE_CTA and YB_CONV_NO_TAIL_SPLIT keep the
 * one-CTA plan.  Pure host logic. */
int yb_conv_config(const yb_op_desc* op, yb_conv_info* info);

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

/* Test-time augmentation (YOLOv5's `augment=True`, yolort/v5/models/yolo.py:152-208): the head logits of up to
 * YB_TTA_MAX_PASSES plan runs over rescaled / mirrored canvases decoded into ONE candidate arena per image and
 * suppressed together.  A pass lists the level slices that take part, in order (the reference's _clip_augmented drops
 * the last level of pass 0 and the first level of pass 2: leave those out).  Every box is decoded, then
 * (cx, cy, w, h) /= scale (fp32 division) and, for a mirrored pass, cx = canvas_w - cx, then converted to corners.
 * Candidate index = (kept anchor over all passes in the order given) * n_classes + class; it must fit 32 bits.
 * The levels must be the plan's NHWC head buffers (16-bit logits, rows of <= 512 bytes).  `p->n_levels` is not read.
 * Outputs, status words and the overflow rule are those of yb_decode_nms. */
#define YB_TTA_MAX_PASSES 3
typedef struct {
  int32_t n_levels;        /* level slices of this pass that take part (<= YB_MAX_LEVELS)            */
  int32_t flip_lr;         /* 1: the pass ran on the left-right mirrored canvas                      */
  float scale;             /* the pass's canvas scale s                                              */
  float canvas_w;          /* Wb, width of the unscaled canvas (un-mirroring: cx = Wb - cx)          */
  yb_head_level levels[YB_MAX_LEVELS];
} yb_tta_pass;
size_t yb_decode_nms_tta_workspace_bytes(const yb_nms_params* p, int n_passes, const yb_tta_pass* passes);
int yb_decode_nms_tta(const yb_nms_params* p, int n_passes, const yb_tta_pass* passes, const float* rescale_dev,
                      float* boxes_dev, float* scores_dev, int64_t* labels_dev, int32_t* counts_dev, int64_t* status_dev,
                      void* workspace_dev, size_t workspace_bytes, void* stream);

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

/* ------------------------------------------------------------------------------------------------
 * Baseline JPEG decode  (replaces the reference's default loader `read_image(path, mode=RGB)`,
 * yolort/models/yolov5.py:218-228, for the files it can take; bit-identical to that CPU decoder:
 * libjpeg's islow IDCT, "fancy" upsampling and integer YCbCr->RGB)
 * Subset: SOF0/SOF1, 8-bit, Huffman, one interleaved scan holding every component; 1 component (gray,
 * replicated to RGB) or 3 components libjpeg reads as YCbCr; per-component sampling ratios 1x1, 2x1
 * (4:2:2) and 2x2 (4:2:0); restart intervals; APPn / COM skipped.  Anything else is reported as
 * unsupported by yb_jpeg_parse, with the reason.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t supported;           /* 1: yb_jpeg_decode takes this file; 0: `reason` says why not            */
  char reason[92];
  int32_t width, height;
  int32_t ncomp;               /* 1 or 3                                                                  */
  int32_t h_samp[3], v_samp[3];
  int32_t restart_interval;    /* MCUs per restart interval, 0 = no DRI                                  */
  int32_t mcus_x, mcus_y, blocks_per_mcu;
  int64_t scan_begin, scan_end; /* the entropy-coded segment: file bytes [scan_begin, scan_end)           */
  int64_t data_offset;         /* set by the caller: where byte 0 of the file lies in yb_jpeg_decode's src */
  uint16_t quant[3][64];       /* per component, natural (row-major) order                               */
  uint8_t dc_bits[3][16], ac_bits[3][16]; /* per component: number of codes of length 1..16             */
  uint8_t dc_vals[3][16];
  uint8_t ac_vals[3][256];
} yb_jpeg_info;

/* status bits of yb_jpeg_decode, per image (0 = decoded cleanly) */
#define YB_JPEG_ST_HUFFMAN 1   /* a bit pattern that is no code of its table                             */
#define YB_JPEG_ST_COEF 2      /* a run that moves the coefficient index past 63                          */
#define YB_JPEG_ST_TRUNCATED 4 /* the data ends before the last MCU, an interval holds the wrong number of
                                  MCUs, or data follows the last MCU                                      */
#define YB_JPEG_ST_RESTART 8   /* a restart marker out of sequence, missing or unexpected                 */
#define YB_JPEG_ST_RANGE 16    /* an IDCT value outside [-512, 511] (or a 16-bit overflow): libjpeg's C and
                                  SIMD code disagree there, so the CPU decoder is the one to ask          */

/* Host-only: reads the markers of `data` (nothing in it is trusted: every length and table is checked)
 * and fills `info`.  Returns YB_OK for any input; info->supported says whether the device decoder takes it. */
int yb_jpeg_parse(const uint8_t* data, int64_t len, yb_jpeg_info* info);

/* Host-only: workspace yb_jpeg_decode needs for these images (all of them supported). */
size_t yb_jpeg_workspace_bytes(int n, const yb_jpeg_info* infos);

/* Decodes n files on `stream` without a host synchronisation.  `infos` (host) are yb_jpeg_parse results with
 * data_offset filled in; `src_dev` starts with a copy of infos[0..n) (n * sizeof(yb_jpeg_info) bytes, so one
 * host-to-device copy carries tables and compressed bytes together) and holds file i at src_dev +
 * infos[i].data_offset.  dst_dev[i] (a host array of device pointers) receives image i as HWC uint8 RGB,
 * height x width x 3, rows packed.  status_dev: int32[n], YB_JPEG_ST_* bits per image; a nonzero image's pixels
 * are undefined.  The kernels touch no byte of dst outside each image's extent. */
int yb_jpeg_decode(int n, const yb_jpeg_info* infos, const void* src_dev, uint8_t* const* dst_dev,
                   int32_t* status_dev, void* workspace_dev, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * COCO box evaluation  (replaces pycocotools' COCOeval.evaluate + accumulate behind the reference's
 * COCOEvaluator, yolort/data/coco_eval.py:28-217, iouType "bbox"; the protocol is restated rule by rule in
 * oracle/restate_cocoeval.py and reproduced bit for bit)
 * ---------------------------------------------------------------------------------------------- */
typedef struct {               /* host struct of device pointers, uploaded once per annotation file          */
  int32_t n_images;            /* image index i = the i-th smallest image id of the file                      */
  int32_t n_categories;        /* K; category index k = the k-th smallest category id                         */
  int32_t n_gt;                /* annotations                                                                 */
  int32_t max_gt_per_pair;     /* most annotations of one (image, category)                                   */
  const int32_t* img_start;    /* [n_images+1]: the annotations of image i are [img_start[i], img_start[i+1])  */
  const int32_t* gt_img;       /* [n_gt] image index                                                          */
  const int32_t* gt_cat;       /* [n_gt] category index: ascending within an image, file order within a pair  */
  const double* gt_box;        /* [n_gt][4] x, y, w, h as in the file (16-byte aligned)                       */
  const double* gt_area;       /* [n_gt] the annotation's `area` field                                        */
  const uint8_t* gt_flags;     /* [n_gt] YB_COCO_GT_* bits                                                    */
} yb_coco_gt;

#define YB_COCO_GT_CROWD 1          /* iscrowd != 0: ignored, and its IoU's union is the detection's area      */
#define YB_COCO_GT_ID_NONZERO 2     /* a match to an annotation whose id is 0 counts as no match               */
#define YB_COCO_ST_UNKNOWN_IMAGE 1  /* status bit: a detection on an image the file does not have             */
#define YB_COCO_ST_BAD_LABEL 2      /* status bit: a label outside the label map                               */
#define YB_COCO_ROW_DROPPED (-2)    /* row_image value: skip the row (its image was evaluated before)          */
#define YB_COCO_RECORD_INT32 8      /* one stored detection: image, position, category (-1: not evaluated),
                                       score bits, then x, y, w, h as fp32 bits                               */
#define YB_COCO_NUM_PARAMS 119      /* float64 iouThrs[10] | recThrs[101] | areaRng[4][2]                     */

/* Appends an n x d padded batch (forward_padded's layout: boxes xyxy fp32 [n,d,4], scores fp32 [n,d], labels
 * int64 [n,d], counts int32 [n]) as n*d records at records_dev (16-byte aligned).  row_image_dev: int32 [n],
 * the image index of each row, -1 for an image id the file does not have, or YB_COCO_ROW_DROPPED.
 * label_map_dev: int32 [n_labels], label -> category index, -1 for a category the file does not have.  Slots
 * at or past counts[row] are stored as not evaluated.  Errors found in the data are ORed into *status_dev
 * (YB_COCO_ST_*).  No host synchronisation. */
int yb_coco_append(int n, int d, const float* boxes_dev, const float* scores_dev, const int64_t* labels_dev,
                   const int32_t* counts_dev, const int32_t* row_image_dev, const int32_t* label_map_dev,
                   int32_t n_labels, int32_t* records_dev, int32_t* status_dev, void* stream);

/* Host-only: workspace yb_coco_evaluate needs for n_records records against `gt`. */
size_t yb_coco_evaluate_workspace_bytes(int64_t n_records, const yb_coco_gt* gt);

/* Evaluates the stored records against `gt` over the images with evaluated_dev[i] != 0 (uint8 [n_images]; every
 * record must lie on such an image).  params_dev: YB_COCO_NUM_PARAMS float64 values.  Writes COCOeval.eval's
 * arrays as float64: precision_dev and scores_dev [10][101][K][4][3], recall_dev [10][K][4][3], -1 where
 * pycocotools leaves -1.  No host synchronisation. */
int yb_coco_evaluate(const yb_coco_gt* gt, const int32_t* records_dev, int64_t n_records, const uint8_t* evaluated_dev,
                     const double* params_dev, double* precision_dev, double* recall_dev, double* scores_dev,
                     void* workspace_dev, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * YOLOv5 training loss  (the reference's SetCriterion, yolort/models/box_head.py:85-325: target assignment
 * :233-325, CIoU box loss :190-195 with yolort/models/_utils.py:26-40 / :65-108, objectness :197-217, class
 * loss :205-212, gains :223-225; restated rule by rule in oracle/restate_loss.py)
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  const void* logits;          /* head output [N, A, H, W, K], contiguous, K = n_classes + 5                   */
  int32_t dtype;               /* YB_F32 / YB_F16 / YB_BF16                                                   */
  int32_t H, W;                /* the level's grid (the gain of box_head.py:271 is W, H, W, H)                 */
  float stride_px;             /* anchors are divided by it in fp32 (box_head.py:167-171)                      */
  float anchors_px[2 * YB_MAX_ANCHORS];  /* (w, h) per anchor in pixels                                       */
} yb_loss_level;

typedef struct {
  int32_t n_images, n_levels, n_anchors, n_classes;  /* N, L <= YB_MAX_LEVELS, A <= YB_MAX_ANCHORS, nc       */
  float box_gain, cls_gain, obj_gain;  /* box_head.py:223-225                                                 */
  float cls_pos, obj_pos;      /* BCE pos_weight of the class and objectness terms (:175-176)                  */
  float anchor_thresh;         /* ratio test max(r, 1/r) < anchor_thresh, compared in fp32 (:278)              */
  float smooth_pos, smooth_neg;  /* class targets (:140-141, _utils.py:111-114)                               */
  float gr;                    /* objectness target (1 - gr) + gr * clamp(CIoU, 0) (:203)                      */
  float balance[YB_MAX_LEVELS];  /* objectness weight per level (:217)                                        */
} yb_yolo_loss_params;

#define YB_LOSS_ST_IMAGE 1          /* status bit: a target's image index is outside [0, N)                  */
#define YB_LOSS_ST_CLASS 2          /* status bit: a target's class is outside [0, nc)                        */
#define YB_LOSS_ST_NONFINITE 4      /* status bit: a target's cx, cy, w or h is not finite                    */
#define YB_LOSS_MATCH_INT32 24      /* one match record: level, b, a, gj, gi, class, cell, 0, tbox[4] (fp32),
                                       anchor[2] (fp32, grid units), objectness target, 1 - CIoU, then
                                       d box loss / d logit[4] and the class BCE sum (fp32), 3 unused words   */

/* Host-only: workspace the loss needs for n_targets targets over these levels (0 for an invalid request). */
size_t yb_yolo_loss_workspace_bytes(const yb_yolo_loss_params* params, const yb_loss_level* levels,
                                    int64_t n_targets);

/* Host-only: where the matches live in the workspace.  out[0] = byte offset of the match records
 * (YB_LOSS_MATCH_INT32 words each, ordered level, then offset, anchor, target as box_head.py:297 does),
 * out[1] = byte offset of the int32 match counts: element l * 5 * A * n_targets is the index of level l's first
 * match, element n_levels * 5 * A * n_targets the total.  out[2] = the record capacity. */
int yb_yolo_loss_layout(const yb_yolo_loss_params* params, const yb_loss_level* levels, int64_t n_targets,
                        int64_t* out);

/* Forward.  targets_dev: fp32 [n_targets, 6] (image, class, cx, cy, w, h), normalised to the canvas.  Writes
 * out_losses_dev: fp32 [3 + n_levels] = loss_cls, loss_box, loss_obj (gains applied) and each level's
 * objectness mean before its balance.  Invalid targets OR YB_LOSS_ST_* bits into *status_dev and take no part; no
 * thread reads outside the arrays.  No host synchronisation, no float atomics: a repeated call gives the same bits.
 * The workspace keeps what yb_yolo_loss_backward needs. */
int yb_yolo_loss_forward(const yb_yolo_loss_params* params, const yb_loss_level* levels, const float* targets_dev,
                         int64_t n_targets, float* out_losses_dev, int32_t* status_dev, void* workspace_dev,
                         size_t workspace_bytes, void* stream);

/* Backward of the forward call that filled `workspace_dev` (same params, levels and n_targets).  grad_losses_dev:
 * fp32 [3], the incoming gradients of loss_cls, loss_box, loss_obj.  grad_out_levels[l] (host array of device
 * pointers) receives d loss / d logits of level l, in that level's dtype and layout, every element written once,
 * computed in fp32 and rounded once.  Matches that share a cell are summed in match order. */
int yb_yolo_loss_backward(const yb_yolo_loss_params* params, const yb_loss_level* levels, int64_t n_targets,
                          const float* grad_losses_dev, void* const* grad_out_levels, void* workspace_dev,
                          size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Weight gradient of 1x1 convolutions  (the backward of the detection head's nn.Conv2d layers,
 * yolort/models/box_head.py:35-37,68-82, with respect to weight and bias)
 *   dW[co][ci] = sum_p dY[p][co] * X[p][ci]      db[co] = sum_p dY[p][co]
 * over the P = N*H*W pixels of NHWC rows.  Sums are fp32 in a fixed order (split-K partial tiles in the workspace,
 * then an ordered reduction), rounded once to out_dtype; no float atomics, so a repeated call on the same device gives
 * the same bits.  Up to YB_WGRAD_MAX_PROBLEMS problems (e.g. the levels of a head) share one launch pair.
 * ---------------------------------------------------------------------------------------------- */
#define YB_WGRAD_MAX_PROBLEMS 8

typedef struct {
  int32_t dtype;               /* YB_F16 / YB_BF16: dy and x (every problem of a call has the same)            */
  int32_t out_dtype;           /* YB_F32 / YB_F16 / YB_BF16: dw and db                                          */
  int64_t P;                   /* pixels (rows of dy and x), 1 <= P < 2^31                                      */
  int32_t Cout, Cin;           /* dw is [Cout][Cin] row-major (the nn.Conv2d weight [Cout, Cin, 1, 1])          */
  const void* dy;              /* [P][dy_stride], 16-byte aligned; Cout <= dy_stride, dy_stride % 8 == 0        */
  int64_t dy_stride;
  const void* x;               /* [P][x_stride], 16-byte aligned; Cin <= x_stride, x_stride % 8 == 0            */
  int64_t x_stride;
  void* dw;                    /* [Cout][Cin], aligned to its element size                                      */
  void* db;                    /* optional [Cout], may be NULL                                                  */
} yb_wgrad_problem;

/* Host-only: workspace bytes yb_conv_wgrad needs for these problems (0 for an invalid request). */
size_t yb_conv_wgrad_workspace_bytes(const yb_wgrad_problem* problems, int n);

/* Host-only introspection of the launch (tests, tuning).  `info` receives 8 + 4 * n ints:
 *   [0] work items (CTA tiles)  [1] grid  [2] dynamic shared memory  [3] pipeline stages  [4] pixels per stage
 *   [5] output rows per tile  [6] maximum input channels per tile  [7] blocks of 256 outputs in the reduction
 *   then per problem q at 8 + 4q: output-row tiles, input-channel tiles, pixel slices, pixels per slice.
 * Slice s of problem q covers pixels [s * len, min((s + 1) * len, P)); every slice is non-empty. */
int yb_conv_wgrad_config(const yb_wgrad_problem* problems, int n, int32_t* info);

/* Enqueues the partial-tile launch and the reduction launch on `stream`.  No host synchronisation, no allocation.
 * Argument errors return YB_ERR_INVALID before anything touches the device; a workspace smaller than
 * yb_conv_wgrad_workspace_bytes returns YB_ERR_WORKSPACE. */
int yb_conv_wgrad(const yb_wgrad_problem* problems, int n, void* workspace_dev, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training augmentations (the reference's yolort/data/transforms.py:21-336 on uint8 tensor images, with
 * torchvision's tensor arithmetic; restated in oracle/restate_augment.py).  Each image carries its recipe: the ops
 * its transforms drew, in call order.  Every parameter is drawn on the host; the kernels only compute pixels.
 * ---------------------------------------------------------------------------------------------- */
#define YB_AUG_MAX_OPS 16
#define YB_AUG_MAX_CONTRAST 4      /* contrast ops per image (one mean launch each)                          */
#define YB_AUG_BRIGHTNESS 1        /* factor, one_minus                                                      */
#define YB_AUG_CONTRAST 2          /* factor, one_minus; arg = round, h, w of the image the op sees          */
#define YB_AUG_SATURATION 3        /* factor, one_minus                                                      */
#define YB_AUG_HUE 4               /* factor                                                                 */
#define YB_AUG_PERMUTE 5           /* arg = source channel of output channel 0, 1, 2                         */
#define YB_AUG_ZOOM_OUT 6          /* arg = top, left, h, w of the image on the canvas, canvas h, w,
                                      fill (r | g<<8 | b<<16)                                                */
#define YB_AUG_CROP 7              /* arg = top, left, h, w of the window                                    */
#define YB_AUG_HFLIP 8             /* arg = width                                                            */

typedef struct {
  int32_t kind;                /* YB_AUG_*                                                                    */
  int32_t arg[7];
  float factor;                /* the drawn factor (an fp32 value)                                            */
  float one_minus;             /* 1.0 - factor computed in double, rounded to fp32 (torchvision's _blend)      */
} yb_aug_op;

typedef struct {
  const uint8_t* src;          /* uint8 [3, src_h, src_w] with these element strides                          */
  int64_t stride_c, stride_y, stride_x;
  int32_t src_h, src_w, out_h, out_w;
  int64_t out_offset;          /* elements from the output base to this image's contiguous [3, out_h, out_w]   */
  int32_t n_ops, n_contrast;
  int32_t out_block_start;     /* filled by yb_augment_prepare                                                */
  int32_t mean_block_start[YB_AUG_MAX_CONTRAST];
  int32_t reserved;
  yb_aug_op ops[YB_AUG_MAX_OPS];
} yb_aug_image;

/* Host-only: checks the recipes (out_h / out_w and each contrast op's h, w must be the sizes the ops give; crops
 * lie inside their image) and fills n_contrast and the block starts.  totals[0] = output blocks, totals[1 + j] =
 * blocks of mean round j, for YB_AUG_MAX_CONTRAST rounds. */
int yb_augment_prepare(int n_images, yb_aug_image* images, int64_t* totals);

/* Computes every image's output.  images_host: the prepared descriptors; images_dev: the same bytes on the device.
 * out_dtype YB_U8, or YB_F32 for the fused byte / 255.0f (IEEE division).  sums_dev: uint64
 * [n_images * YB_AUG_MAX_CONTRAST], the exact grayscale sums of the contrast ops (zeroed here).  One mean launch per
 * contrast round that any image has, then one output launch.  No host synchronisation; deterministic. */
int yb_augment(int n_images, const yb_aug_image* images_host, const yb_aug_image* images_dev, void* out_dev,
               int32_t out_dtype, uint64_t* sums_dev, void* stream);

/* The device parameter sampler (Compose.apply_batch(..., generator=)): the transforms of a Compose, each drawn from
 * Philox4x32-10 with key = the call's 64-bit draw and counter = (image, transform index, a, b).  The rules are
 * restated in oracle/sample_augment.py. */
#define YB_AUG_MAX_TRANSFORMS 16
#define YB_AUG_MAX_OPTIONS 16
#define YB_AUG_CROP_ROUNDS 1024    /* IoU-crop rounds before an image gives up                               */
#define YB_AUG_S_NONE 0            /* PILToTensor, ConvertImageDtype: no draw                                */
#define YB_AUG_S_PHOTOMETRIC 1     /* p; jitter bit j: range j (brightness, contrast, saturation, hue) drawn  */
#define YB_AUG_S_ZOOM_OUT 2        /* p; range 0 = side range; fill                                          */
#define YB_AUG_S_IOU_CROP 3        /* range 0 = scale; aspect bounds; options; trials                        */
#define YB_AUG_S_HFLIP 4           /* p                                                                      */
#define YB_AUG_ST_CROP_ROUNDS 1    /* status: an IoU crop accepted no window in YB_AUG_CROP_ROUNDS rounds   */

typedef struct {
  int32_t kind;                /* YB_AUG_S_*                                                                  */
  int32_t jitter;
  int32_t trials, n_options;
  uint32_t fill;               /* r | g<<8 | b<<16                                                            */
  float p;                     /* a transform applies when its uniform is below p                             */
  float lo[4], span[4];        /* a value drawn from a range is lo + u * span in fp32                         */
  double min_aspect, max_aspect;
  double options[YB_AUG_MAX_OPTIONS];
} yb_aug_sampler;

/* Draws every image's recipe on the device: one warp per image.  transforms: host array (it travels as a kernel
 * argument).  key_dev: int64 [2], the key's words are their low 32 bits.  descs_dev: src_h, src_w read, n_ops, ops,
 * out_h and out_w written as the host sampler fills them.  Image i's boxes (fp32 [n, 4] xyxy) and labels (int64) are
 * rows [box_start[i], box_start[i + 1]) of boxes_dev / labels_dev; its kept boxes go to the same rows of boxes_out_dev
 * / labels_out_dev in order, their number to counts_dev[i], YB_AUG_ST_* bits to status_dev[i].  The box pointers may
 * be null when the batch has no boxes.  No host synchronisation, no float atomics: a repeated call writes the same
 * bits.  Argument errors return YB_ERR_INVALID before the device is touched. */
int yb_augment_sample(int n_images, const yb_aug_sampler* transforms, int n_transforms, const int64_t* key_dev,
                      yb_aug_image* descs_dev, const float* boxes_dev, const int64_t* labels_dev,
                      const int32_t* box_start_dev, float* boxes_out_dev, int64_t* labels_out_dev, int32_t* counts_dev,
                      int32_t* status_dev, void* stream);

/* YOLOv5's own augmentations (yolort/v5/utils/augmentations.py) on uint8 [H, W, 3] images, OpenCV's arithmetic:
 * csrc/v5_augment.cu, restated in oracle/restate_v5aug.py.  An output pixel maps back through the flips, then
 * through the inverse warp (OpenCV's fixed-point bilinear remap, border 114), then runs BGR->HSV, the image's LUT and
 * HSV->BGR, then the last cutout rectangle holding it sets its value.  Each step runs when its bit is set. */
#define YB_V5_MAX_RECTS 31
#define YB_V5_AFFINE 1          /* warp: inv[0..5] is warpAffine's inverse 2x3 map                             */
#define YB_V5_PERSPECTIVE 2     /* warp: inv[0..8] is warpPerspective's inverse 3x3 map                        */
#define YB_V5_TO_HSV 4          /* COLOR_BGR2HSV (COLOR_RGB2HSV with YB_V5_RGB)                                */
#define YB_V5_LUT 8             /* channel c <- lut[c][channel c]                                              */
#define YB_V5_FROM_HSV 16       /* COLOR_HSV2BGR (COLOR_HSV2RGB with YB_V5_RGB)                                */
#define YB_V5_RGB 32            /* the image holds r, g, b: the colour steps swap b and r                      */
#define YB_V5_FLIP_LR 64        /* the output is mirrored left-right (np.fliplr) after the colour steps        */
#define YB_V5_FLIP_UD 128       /* the output is mirrored up-down (np.flipud) after the colour steps           */

typedef struct {
  const uint8_t* src;          /* [src_h, src_w, 3] with element strides                                      */
  uint8_t* dst;                /* [out_h, out_w, 3] with element strides; may be src when no warp or flip bit  */
  int64_t src_stride_y, src_stride_x, src_stride_c;
  int64_t dst_stride_y, dst_stride_x, dst_stride_c;
  int32_t src_h, src_w, out_h, out_w;
  int32_t ops;                 /* YB_V5_* bits                                                                */
  int32_t n_rects;             /* cutout rectangles, applied in order                                         */
  int32_t block_start;         /* filled by yb_v5_augment_prepare: the image's first block                    */
  int32_t reserved;
  double inv[9];
  int32_t rects[YB_V5_MAX_RECTS][4];   /* y0, x0, y1, x1 (half-open) in output pixels                          */
  uint32_t rect_color[YB_V5_MAX_RECTS];  /* c0 | c1<<8 | c2<<16, in the image's channel order               */
  uint8_t lut[3][256];
} yb_v5_image;

/* Host-only: checks the descriptors and fills block_start; *total_blocks = the launch's blocks. */
int yb_v5_augment_prepare(int n_images, yb_v5_image* images, int64_t* total_blocks);

/* Computes every image in one launch.  images_dev: the prepared descriptors on the device.  No host
 * synchronisation; a repeated call writes the same bits. */
int yb_v5_augment(int n_images, const yb_v5_image* images_dev, int64_t total_blocks, void* stream);

/* mixup: dst[i] = uint8(trunc(a[i] * r + b[i] * (1 - r))) in IEEE double, over n contiguous bytes. */
int yb_v5_mixup(const uint8_t* a_dev, const uint8_t* b_dev, uint8_t* dst_dev, int64_t n, double r, void* stream);

/* YOLOv5's mosaic training batches (the augment=True, rect=False branch of upstream v6.0's
 * LoadImagesAndLabels.__getitem__: load_image, load_mosaic or letterbox, random_perspective, mixup, augment_hsv, the
 * flips; yolort_b200/v5/utils/datasets.py draws every parameter).  Two launches:
 *
 * yb_v5_resize: load_image's cv2.resize(INTER_LINEAR) of uint8 [H, W, 3] images, OpenCV 4.x's 8-bit fixed-point
 * arithmetic (11-bit coefficients, horizontal then vertical pass, the vertical pass in the (S >> 4) * b >> 16 form of
 * VResizeLinearVec_32s8u), and its INTER_AREA average for an exact 2x downscale. */
typedef struct {
  const uint8_t* src;          /* [src_h, src_w, 3] with element strides                                      */
  uint8_t* dst;                /* dense [dst_h, dst_w, 3]                                                     */
  int64_t src_stride_y, src_stride_x, src_stride_c;
  int32_t src_h, src_w, dst_h, dst_w;
  int32_t block_start;         /* filled by yb_v5_resize_prepare: the job's first block                       */
  int32_t reserved;
} yb_v5_resize_job;

/* Host-only: checks the jobs and fills block_start; *total_blocks = the launch's blocks. */
int yb_v5_resize_prepare(int n_jobs, yb_v5_resize_job* jobs, int64_t* total_blocks);

/* Resizes every job in one launch.  jobs_dev: the prepared jobs on the device.  No job may read another's dst. */
int yb_v5_resize(int n_jobs, const yb_v5_resize_job* jobs_dev, int64_t total_blocks, void* stream);

/* yb_v5_resize_area: load_image's cv2.resize(INTER_AREA) (augment=False, the validation loader) of uint8 [H, W, 3]
 * images whose output is no larger than the source on either axis, OpenCV 4.x's 8-bit arithmetic.  Integer factors
 * (both scales within DBL_EPSILON of an integer): 2 x 2 is (sum + 2) >> 2, any other ix x iy
 * cvRound(float(sum) * (1.f / (ix * iy))).  Otherwise computeResizeAreaTab's taps (in double, each weight rounded once
 * to float) and ResizeArea_Invoker's float accumulation order.  Same jobs as yb_v5_resize; a launch of its own. */
int yb_v5_resize_area_prepare(int n_jobs, yb_v5_resize_job* jobs, int64_t* total_blocks);
int yb_v5_resize_area(int n_jobs, const yb_v5_resize_job* jobs_dev, int64_t total_blocks, void* stream);

/* yb_v5_compose: one training sample per descriptor.  The warp reads a virtual canvas: up to YB_V5_MAX_PLACES
 * rectangles, each a view of a (resized) image placed at an offset, and the value 114 everywhere else; the canvas
 * itself is never written.  An output pixel maps back through the flips, then through each canvas's warp (or reads
 * the canvas at the same place), blends the two canvases of a mixup in IEEE double, runs the colour steps and stores
 * channel k at dst + y * dst_stride_y + x * dst_stride_x + k * dst_stride_c (a negative dst_stride_c reverses the
 * channels: CHW RGB from a BGR sample). */
#define YB_V5_MAX_PLACES 4

typedef struct {
  const uint8_t* src;          /* [h, w, 3] with element strides                                             */
  int64_t stride_y, stride_x, stride_c;
  int32_t y0, x0, y1, x1;      /* the canvas rectangle [y0, y1) x [x0, x1) it covers                          */
  int32_t oy, ox;              /* canvas pixel (y, x) of the rectangle is src[y - oy, x - ox]                 */
} yb_v5_place;

typedef struct {
  double inv[9];               /* inverse map, as yb_v5_image's                                               */
  int32_t warp;                /* 0 (no warp: the output is the canvas), YB_V5_AFFINE or YB_V5_PERSPECTIVE     */
  int32_t n_places;            /* 0..YB_V5_MAX_PLACES, disjoint rectangles                                    */
  yb_v5_place places[YB_V5_MAX_PLACES];
} yb_v5_canvas;

typedef struct {
  uint8_t* dst;
  int64_t dst_stride_y, dst_stride_x, dst_stride_c;
  int32_t out_h, out_w;        /* the same for every sample of a launch                                       */
  int32_t ops;                 /* YB_V5_TO_HSV, _LUT, _FROM_HSV, _RGB, _FLIP_LR, _FLIP_UD                      */
  int32_t n_canvases;          /* 1, or 2: mixup of canvas 0 (ratio mix_r) and canvas 1 (1 - mix_r)           */
  double mix_r, mix_omr;       /* r and 1 - r as numpy computes it                                            */
  yb_v5_canvas canvas[2];
  uint8_t lut[3][256];
} yb_v5_sample;

/* Host-only: checks the descriptors; *blocks_per_sample = the launch's blocks per sample. */
int yb_v5_compose_prepare(int n_samples, const yb_v5_sample* samples, int64_t* blocks_per_sample);

/* Computes every sample in one launch.  samples_dev: the descriptors on the device.  No host synchronisation; a
 * repeated call writes the same bits. */
int yb_v5_compose(int n_samples, const yb_v5_sample* samples_dev, int64_t blocks_per_sample, void* stream);

/* YOLOv5's validation rescale (val.py v6.0): predictions and labels of one rect batch back to each image's native
 * pixels, in torch's CPU float32 arithmetic (on CUDA tensors torch multiplies by the float reciprocal of gain
 * instead, which can differ by one unit in the last place).  A box goes through scale_coords(..., ratio_pad) and clip_coords: x - pad_w, y - pad_h, each
 * divided by gain with correct rounding, then x clamped to [0, w0] and y to [0, h0] (NaN kept, as torch.clamp keeps it).  A target row (image, cls, x, y, w, h)
 * normalised is first multiplied by (canvas_w, canvas_h) and turned into xyxy (xywh2xyxy, w / 2 as w * 0.5); it is
 * written to targets_out, and one whose image index is not an integer in [0, n) is only converted.  One launch, no
 * host synchronisation. */
typedef struct {
  float* boxes;                /* [n, D, 4] xyxy, in place; slots d >= counts[i] are not touched              */
  const int32_t* counts;       /* [n]                                                                         */
  const float* targets;        /* [T, 6] (image, cls, x, y, w, h) normalised to the canvas                    */
  float* targets_out;          /* [T, 6] (image, cls, x1, y1, x2, y2) native pixels; may be targets            */
  const float* params;         /* [n, 5] per image: gain, pad_w, pad_h, h0, w0                                */
  int32_t n, D;
  int64_t T;
  float canvas_w, canvas_h;
} yb_v5_rescale;

int yb_v5_rescale_coords(const yb_v5_rescale* r, void* stream);

/* YOLOv5's AutoAnchor (yolort/v5/utils/autoanchor.py; yolort_b200/v5/utils/autoanchor.py draws every random number on
 * the host): csrc/autoanchor.cu, restated in oracle/restate_autoanchor.py.  Labels are float32 (w, h) pairs. */
#define YB_AA_MAX_ANCHORS 64
#define YB_AA_METRIC_WORKSPACE 65536

/* The ratio metric of n labels against n_anchors (w, h) anchors: x = min(r, 1 / r) over both sides, r = label / anchor,
 * best = max over the anchors.  f64 = 0: in float32 (the anchors hold float32 values), the threshold compared as float32;
 * f64 = 1: in float64.  counts_dev[2] = {labels with best > thr, (label, anchor) pairs with x > thr};
 * sums_dev[3] = {sum x, sum best, sum of x > thr} in float64, added in a fixed order.  workspace: YB_AA_METRIC_WORKSPACE
 * bytes of device memory. */
int yb_anchor_metric(const float* wh_dev, int64_t n, const double* anchors_dev, int n_anchors, int f64, double thr,
                     int64_t* counts_dev, double* sums_dev, void* workspace, size_t workspace_bytes, void* stream);

/* Device bytes yb_kmeans needs for n_obs observations, k codes and `trials` trials (0: invalid). */
size_t yb_kmeans_workspace_bytes(int64_t n_obs, int k, int trials);

/* scipy.cluster.vq.kmeans's trials (_kmeans from each starting book guess_dev[trials, k, 2]) over the float64 (x, y)
 * observations, all trials at once, bit for bit.  Outputs per trial: books_dev[trials, k, 2] (the first sizes_dev[t]
 * rows hold the final book), dist_dev[trials] (the final mean distortion); *iters: iterations launched.  The host
 * reads a device count of live trials every check_every iterations and never otherwise waits. */
int yb_kmeans(const double* obs_dev, int64_t n_obs, int k, int trials, const double* guess_dev, double thresh,
              int check_every, double* books_dev, int32_t* sizes_dev, double* dist_dev, int32_t* iters,
              void* workspace, size_t workspace_bytes, void* stream);

/* kmean_anchors' genetic evolution, `gen` generations in one cooperative launch.  k0_dev[n_anchors, 2]: the starting
 * anchors (float64); v_dev[gen, n_anchors, 2]: the mutation factors drawn on the host.  Generation g evaluates
 * kg = max(k * v[g], 2) in float64, its float32 fitness fl32(fl32(S) / n) with S the exact sum of the labels' best
 * ratios above thr (float32 arithmetic), and keeps kg when the fitness is larger.  unit_exp: floor(log2(thr)) - 23,
 * the fixed-point unit of that sum.  Outputs: fit_dev[gen + 1] (the fitness after each generation, [0]: the start),
 * accepted_dev[gen] (1 where kg was kept), k_out_dev[n_anchors, 2].  workspace: (gen + 1) * 8 bytes. */
int yb_anchor_evolve(const float* wh_dev, int64_t n, int n_anchors, const double* k0_dev, const double* v_dev, int gen,
                     double thr, int unit_exp, float* fit_dev, uint8_t* accepted_dev, double* k_out_dev,
                     void* workspace, size_t workspace_bytes, void* stream);

/* YOLOv5's validation metrics (yolort/v5/utils/metrics.py and upstream v6.0 val.py's process_batch):
 * csrc/v5_metrics.cu, restated rule by rule in oracle/restate_v5metrics.py and reproduced bit for bit. */
#define YB_V5M_RECORD_INT32 4            /* one stored detection: conf (float32 bits), class (-1: none), correct bits,
                                            0 (16 bytes: one vector load)                                              */
#define YB_V5M_MAX_IOU 31                /* IoU thresholds: one correct bit each, in a non-negative int32              */
#define YB_V5M_CURVE_POINTS 1000         /* px = np.linspace(0, 1, 1000): the p and r curves                            */
#define YB_V5M_AP_POINTS 101             /* np.linspace(0, 1, 101): compute_ap's interpolation points                  */
#define YB_V5M_NUM_PARAMS 1101           /* float64 px[1000] | x[101], computed by numpy on the host                    */
#define YB_V5M_ST_BAD_IMAGE 1            /* status bit: a target's image index is not an integer in [0, n)             */
#define YB_V5M_ST_BAD_TARGET_CLASS 2     /* status bit: a target's class is not an integer in [0, nc)                  */
#define YB_V5M_ST_BAD_DET_CLASS 4        /* status bit: a detection's class is not an integer in [0, nc)               */
#define YB_V5M_ST_BAD_COUNT 8            /* status bit: a row's detection count is outside [0, d]                      */
#define YB_V5M_ST_TP_EXCEEDS_LABELS 16   /* status bit: a class has more true positives than labels                    */

/* Device bytes yb_v5m_match needs for n_targets targets. */
size_t yb_v5m_match_workspace_bytes(int n_targets);

/* One launch over n images of a padded batch: boxes_dev [n, d, 4] xyxy, scores_dev [n, d], classes_dev [n, d] (float
 * class values), counts_dev [n] (detections per row), targets_dev [n_targets, 6] = (image, class, x1, y1, x2, y2) in
 * the boxes' coordinate space; order_dev [n_targets]: the targets stably sorted by image; start_dev [n + 1]: each
 * image's first position in that order.  Writes records_dev [n * d, YB_V5M_RECORD_INT32]: val.py's correct bits against
 * iouv_dev[n_iou] (class -1 beyond the row's count, and everywhere when nc == 0).  With nc > 0, adds each target's class
 * to label_count_dev[nc] (if not null) and ConfusionMatrix.process_batch's counts (threshold conf_thr, iou_thr) to
 * matrix_dev[(nc + 1) * (nc + 1)] (if not null), for the rows with targets and, unless cm_empty_rows, detections.
 * Bad input sets YB_V5M_ST_* bits in *status_dev.  No host synchronisation. */
int yb_v5m_match(int n, int d, const float* boxes_dev, const float* scores_dev, const float* classes_dev,
                 const int32_t* counts_dev, const float* targets_dev, int n_targets, const int64_t* order_dev,
                 const int64_t* start_dev, int nc, const float* iouv_dev, int n_iou, float conf_thr, float iou_thr,
                 int cm_empty_rows, int32_t* records_dev, int32_t* label_count_dev, int64_t* matrix_dev, int32_t* status_dev,
                 void* workspace_dev, size_t workspace_bytes, void* stream);

/* Device bytes yb_v5m_ap needs for n_records records and nc classes (0: invalid). */
size_t yb_v5m_ap_workspace_bytes(int64_t n_records, int nc);

/* ap_per_class over stored records (records of a class outside [0, nc) are skipped) with label_count_dev[nc] labels per
 * class: ap_dev [nc, n_iou], and at the first threshold p_dev, r_dev [nc, YB_V5M_CURVE_POINTS], all float64; a class
 * without labels or predictions gets zeros.  params_dev: YB_V5M_NUM_PARAMS float64 values.  Sets
 * YB_V5M_ST_TP_EXCEEDS_LABELS in *status_dev when a class has more true positives than labels.  No host
 * synchronisation. */
int yb_v5m_ap(const int32_t* records_dev, int64_t n_records, int nc, int n_iou, const int32_t* label_count_dev,
              const double* params_dev, double* ap_dev, double* p_dev, double* r_dev, int32_t* status_dev,
              void* workspace_dev, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YOLORT_B200_H */
