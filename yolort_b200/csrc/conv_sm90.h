// Host-side handle of one prepared convolution launch (tensor maps + kernel parameters).
#pragma once
#include <cuda_runtime.h>

#include "../../include/yolort_b200.h"

#include <cuda.h>

namespace yb {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 3x3/s1 halo-patch variant (conv3x3_patch_sm90.cu)
struct PatchConvOp;
bool patch_conv_eligible(const yb_op_desc& d);
int patch_conv_create(const yb_op_desc& d, EncodeTiledFn encode_tiled, PatchConvOp** out);
int patch_conv_configure_check(const yb_op_desc& d, int* info = nullptr);   // host-only validation + tiling (no driver calls)
int patch_conv_launch(const PatchConvOp* op, cudaStream_t stream);
void patch_conv_destroy(PatchConvOp* op);

struct ConvOp;
int conv_op_create(const yb_op_desc& d, ConvOp** out);
int conv_configure_check(const yb_op_desc& d, int* info = nullptr);         // host-only validation + tiling (no driver calls)
int conv_op_launch(const ConvOp* op, cudaStream_t stream);
void conv_op_destroy(ConvOp* op);

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled / cuTensorMapEncodeIm2col from the driver (looked up once)
int encode_tiled_entry(EncodeTiledFn* out);
int encode_im2col_entry(EncodeIm2colFn* out);

// e4m3 convolution and the fp16/bf16 -> e4m3 quantisation op (conv_fp8_sm90.cu)
struct Fp8ConvOp;
int fp8_conv_configure_check(const yb_op_desc& d, int* info = nullptr);   // host-only validation + tiling (no driver calls)
int fp8_conv_op_create(const yb_op_desc& d, Fp8ConvOp** out);
int fp8_conv_op_launch(const Fp8ConvOp* op, cudaStream_t stream);
void fp8_conv_op_destroy(Fp8ConvOp* op);
int quantize_configure_check(const yb_op_desc& d);                         // host-only validation (no driver calls)
int quantize_launch(const yb_op_desc& d, cudaStream_t stream);

// multi-head attention (attention_sm90.cu)
struct AttentionOp;
int attention_configure_check(const yb_op_desc& d);   // host-only validation (no driver calls)
int attention_op_create(const yb_op_desc& d, AttentionOp** out);
int attention_op_launch(const AttentionOp* op, cudaStream_t stream);
void attention_op_destroy(AttentionOp* op);

// MobileNetV3 depthwise convolution and squeeze-excitation (mobilenet_sm90.cu)
int dwconv_configure_check(const yb_op_desc& d);      // host-only validation (no driver calls)
int dwconv_launch(const yb_op_desc& d, cudaStream_t stream);
int se_configure_check(const yb_op_desc& d);          // host-only validation (no driver calls)
int se_launch(const yb_op_desc& d, cudaStream_t stream);

// global average pool of the classifiers (pool_global_sm90.cu)
int avgpool_configure_check(const yb_op_desc& d);     // host-only validation (no driver calls)
int avgpool_launch(const yb_op_desc& d, cudaStream_t stream);

// HBM-bound helpers of the neck (pool_upsample.cu)
int spp_pool_launch(const yb_op_desc& d, cudaStream_t stream);
int upsample2x_launch(const yb_op_desc& d, cudaStream_t stream);
int validate_pool_or_upsample(const yb_op_desc& d);
}  // namespace yb
