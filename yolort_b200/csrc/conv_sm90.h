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

// HBM-bound helpers of the neck (pool_upsample.cu)
int spp_pool_launch(const yb_op_desc& d, cudaStream_t stream);
int upsample2x_launch(const yb_op_desc& d, cudaStream_t stream);
int validate_pool_or_upsample(const yb_op_desc& d);
}  // namespace yb
