// Host-side handles of the prepared launches (tensor maps + kernel parameters) and the plan ops' entry points.
#pragma once
#include "host_sm90.h"

namespace yb {

// One prepared convolution launch, on whichever kernel conv_kernel picks.
struct ConvOp {
  virtual ~ConvOp() = default;
  virtual int launch(cudaStream_t stream) const = 0;
};

// The one choice of a convolution kernel (YB_CONV_KERNEL_*): e4m3 for YB_F8E4M3, else the halo-patch kernel for the
// shapes patch_conv_eligible admits, else 1x1 / im2col.
int conv_kernel(const yb_op_desc& d);
int conv_config(const yb_op_desc& d, yb_conv_info* info);   // host-only validation + tiling (no driver calls)
int conv_create(const yb_op_desc& d, ConvOp** out);

// fp16 / bf16 validation shared by the 1x1 / im2col and halo-patch kernels; 1x1 / im2col kernel (conv_sm90.cu)
int conv_validate(const yb_op_desc& d);
int im2col_conv_config(const yb_op_desc& d, yb_conv_info* info);
int im2col_conv_create(const yb_op_desc& d, ConvOp** out);

// 3x3/s1 halo-patch variant (conv3x3_patch_sm90.cu)
bool patch_conv_eligible(const yb_op_desc& d);
int patch_conv_config(const yb_op_desc& d, yb_conv_info* info);
int patch_conv_create(const yb_op_desc& d, ConvOp** out);

// e4m3 convolution and the fp16/bf16 -> e4m3 quantisation op (conv_fp8_sm90.cu)
int fp8_conv_config(const yb_op_desc& d, yb_conv_info* info);
int fp8_conv_create(const yb_op_desc& d, ConvOp** out);
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
