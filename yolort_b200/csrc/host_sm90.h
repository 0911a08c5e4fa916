// Host helpers of the kernels' launch code: the driver's tensor-map encoders and the tensor maps built with them, the
// N-tile and K-pipeline sizing of the implicit-GEMM convolutions, and launches with programmatic dependent launch.
#pragma once
#include "common.cuh"

namespace yb {

// wgmma N of an output tile: the next power of two >= 16 (weight rows past Cout_pad are zero-filled by the TMA unit, the
// store clips columns past Cout)
inline int mma_n(int n) {
  int c = 16;
  while (c < n) c <<= 1;
  return c;
}

// TMA swizzle of a shared-memory box whose rows are `row_bytes` long: the 32/64/128-byte swizzled rows wgmma reads and the
// epilogues write; rows of 16 bytes (16-column e4m3 output boxes) are not swizzled.
inline CUtensorMapSwizzle swizzle_for_row_bytes(uint64_t row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                             : (row_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled / cuTensorMapEncodeIm2col from the driver (the runtime does not export them), looked up once.
inline int tma_encoders(EncodeTiledFn* tiled, EncodeIm2colFn* im2col) {
  static EncodeTiledFn s_tiled = nullptr;
  static EncodeIm2colFn s_im2col = nullptr;
  if (!s_tiled || !s_im2col) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    YB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    YB_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available from the driver");
    s_tiled = reinterpret_cast<EncodeTiledFn>(fn);
    fn = nullptr;
    YB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres));
    YB_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeIm2col not available from the driver");
    s_im2col = reinterpret_cast<EncodeIm2colFn>(fn);
  }
  *tiled = s_tiled;
  *im2col = s_im2col;
  return YB_OK;
}

inline uint64_t tmap_elem_bytes(CUtensorMapDataType dt) { return dt == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2; }

// Tiled view of a channels-last tensor: dims[0] elements per pixel at a pitch of `pitch` elements, then rank - 1 outer
// dimensions, each dense over the one before (W, H, N of an NHWC map; rows of a matrix), read or written in boxes of
// box[] elements.  Boxes are swizzled to their row bytes.  `what` names the operand in the error.
inline int tmap_tiled(CUtensorMap* map, const char* what, CUtensorMapDataType dt, const void* base, int rank,
                      const cuuint64_t* dims, uint64_t pitch, const cuuint32_t* box, CUtensorMapL2promotion l2) {
  EncodeTiledFn tiled;
  EncodeIm2colFn im2col;
  const int rc = tma_encoders(&tiled, &im2col);
  if (rc != YB_OK) return rc;
  cuuint64_t strides[4];
  strides[0] = pitch * tmap_elem_bytes(dt);
  for (int i = 1; i + 1 < rank; ++i) strides[i] = strides[i - 1] * dims[i];
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult cr = tiled(map, dt, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            swizzle_for_row_bytes(box[0] * tmap_elem_bytes(dt)), l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d", what, static_cast<int>(cr));
    return YB_ERR_CUDA;
  }
  return YB_OK;
}

// Row-major matrix of `rows` rows of `cols` elements at a pitch of `pitch` elements, in boxes of box_rows x box_cols.
inline int tmap_matrix(CUtensorMap* map, const char* what, CUtensorMapDataType dt, const void* base, uint64_t cols,
                       uint64_t rows, uint64_t pitch, uint32_t box_cols, uint32_t box_rows, CUtensorMapL2promotion l2) {
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint32_t box[2] = {box_cols, box_rows};
  return tmap_tiled(map, what, dt, base, 2, dims, pitch, box, l2);
}

// im2col view of the NHWC input of convolution `d`: a load walks box_pixels output pixels of one filter tap and takes
// box_c channels of each; the TMA unit applies padding and stride and zero-fills the halo.
inline int tmap_im2col(CUtensorMap* map, const char* what, CUtensorMapDataType dt, const yb_op_desc& d, uint32_t box_c,
                       uint32_t box_pixels) {
  EncodeTiledFn tiled;
  EncodeIm2colFn im2col;
  const int rc = tma_encoders(&tiled, &im2col);
  if (rc != YB_OK) return rc;
  const uint64_t cs = static_cast<uint64_t>(d.in_cstride) * tmap_elem_bytes(dt);
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(d.W), static_cast<cuuint64_t>(d.H),
                              static_cast<cuuint64_t>(d.N)};
  const cuuint64_t strides[3] = {cs, cs * d.W, cs * d.W * d.H};
  const int lower[2] = {-d.pad, -d.pad};
  const int upper[2] = {d.pad - (d.ksize - 1), d.pad - (d.ksize - 1)};
  const cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(d.stride), static_cast<cuuint32_t>(d.stride), 1};
  const CUresult cr = im2col(map, dt, 4, const_cast<void*>(d.in), dims, strides, lower, upper, box_c, box_pixels, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for_row_bytes(box_c * tmap_elem_bytes(dt)),
                             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeIm2col failed with CUresult %d (Cin=%d cs=%d H=%d W=%d N=%d k=%d s=%d box=%u)", what,
              static_cast<int>(cr), d.Cin, d.in_cstride, d.H, d.W, d.N, d.ksize, d.stride, box_c);
    return YB_ERR_CUDA;
  }
  // Driver workaround also applied by CUTLASS (copy_traits_sm90_im2col.hpp): for tensors smaller than 128 KiB, drivers
  // <= 13.1 set a descriptor bit that makes im2col loads fault.
  int drv = 0;
  cudaDriverGetVersion(&drv);
  if (drv <= 13010 && cs * d.W * d.H * d.N < 131072) reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
  return YB_OK;
}

// Output rows M = N x Ho x Wo of convolution `d`, after checking the output extent against the input, kernel, stride
// and padding.
inline int conv_rows(const yb_op_desc& d, const char* who, int* M) {
  const int Ho = (d.H + 2 * d.pad - d.ksize) / d.stride + 1;
  const int Wo = (d.W + 2 * d.pad - d.ksize) / d.stride + 1;
  YB_REQUIRE(Ho == d.Ho && Wo == d.Wo, "%s: output extent mismatch (%d,%d) vs (%d,%d)", who, Ho, Wo, d.Ho, d.Wo);
  const long long M_ll = static_cast<long long>(d.N) * Ho * Wo;
  YB_REQUIRE(M_ll > 0 && M_ll < (1ll << 31), "%s: M out of range", who);
  *M = static_cast<int>(M_ll);
  return YB_OK;
}

// N tile of the 1x1 / im2col and e4m3 kernels: the whole Cout up to 256 columns (fewest A re-reads); halved when that
// leaves fewer than two 128-row tiles per SM so the persistent grid balances better (not under a chained tail).
inline int conv_block_n(int cout, int m_tiles128, bool chained) {
  const int n_tiles = (cout + 255) / 256;
  int block_n = mma_n((cout + n_tiles - 1) / n_tiles);
  if (m_tiles128 * n_tiles < 2 * num_sms() && block_n > 128 && !chained) block_n /= 2;
  return block_n;
}

// K pipeline of the 1x1 / im2col and e4m3 kernels: `num_k_iters` A sub-tiles of a_bytes (and B sub-tiles of b_bytes)
// per output tile, in stages of kpg sub-tiles.
struct KPipeline {
  int b_resident;        // the weights of the CTA's N tile stay in shared memory
  uint32_t b_res_bytes;
  int kpg;               // k-iterations carried by one stage
  int stages;
  size_t smem;           // dynamic shared memory: stages, resident weights and `fixed`
};

// Weights stay resident when the CTA keeps one N tile (`fixed_n`) and they take at most 80 KB: the persistent CTA then
// streams only activations (halves the L2->SM traffic of the shallow layers).  Stages aim at ~32 KB, so that one mbarrier
// round trip moves enough bytes (a 16-channel tap is only 4 KB), in near-equal groups, with at least three stages in
// flight; as many stages as the rest of `budget` holds, 2 to max_stages.
inline int size_k_pipeline(size_t budget, size_t fixed, uint32_t a_bytes, uint32_t b_bytes, int num_k_iters, bool fixed_n,
                           int max_stages, const char* who, int block_n, KPipeline* kp) {
  const size_t b_total = static_cast<size_t>(num_k_iters) * b_bytes;
  kp->b_resident = (fixed_n && b_total <= 80 * 1024) ? 1 : 0;
  kp->b_res_bytes = kp->b_resident ? static_cast<uint32_t>(b_total) : 0u;
  const uint32_t per_iter = a_bytes + (kp->b_resident ? 0u : b_bytes);
  YB_REQUIRE(budget > fixed + kp->b_res_bytes + 2 * per_iter, "%s: shared memory budget exceeded (block_n=%d)", who, block_n);
  const size_t avail = budget - fixed - kp->b_res_bytes;
  const size_t target = avail / 3 < 32 * 1024 ? avail / 3 : 32 * 1024;
  int kpg_max = static_cast<int>(target / per_iter);
  if (kpg_max < 1) kpg_max = 1;
  if (kpg_max > num_k_iters) kpg_max = num_k_iters;
  const int kgroups = (num_k_iters + kpg_max - 1) / kpg_max;
  kp->kpg = (num_k_iters + kgroups - 1) / kgroups;
  const uint32_t stage_bytes = kp->kpg * per_iter;
  int stages = static_cast<int>(avail / stage_bytes);
  if (stages > max_stages) stages = max_stages;
  if (stages < 2) stages = 2;
  kp->stages = stages;
  kp->smem = static_cast<size_t>(stages) * stage_bytes + kp->b_res_bytes + fixed;
  YB_REQUIRE(kp->smem <= budget, "%s: %zu bytes of shared memory needed, %zu available", who, kp->smem, budget);
  return YB_OK;
}

// Launches `kernel` with programmatic dependent launch: it may start while the previous kernel in the stream drains (its
// griddepcontrol.wait holds it until that kernel's writes are visible).  cluster_x > 1 also groups the CTAs into clusters
// of cluster_x along x.
template <typename... Params, typename... Args>
cudaError_t launch_pdl_cluster(unsigned cluster_x, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem,
                               cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster_x;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cluster_x > 1 ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<Args&&>(args)...);
}

template <typename... Params, typename... Args>
cudaError_t launch_pdl(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  return launch_pdl_cluster(1, kernel, grid, block, smem, stream, static_cast<Args&&>(args)...);
}

}  // namespace yb
