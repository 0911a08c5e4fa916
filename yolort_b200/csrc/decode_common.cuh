// Score-key encoding and reference-order arithmetic shared by the stand-alone decode kernel (decode_nms.cu) and the
// fused decode epilogue of the head convolutions (conv_sm90.cu).
#pragma once
#include "common.cuh"

namespace yb {

__device__ __forceinline__ uint32_t orderable_desc(float f) {
  uint32_t u = __float_as_uint(f);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending order of floats
  return ~u;                                       // descending
}
__device__ __forceinline__ float from_orderable_desc(uint32_t k) {
  uint32_t u = ~k;
  u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
  return __uint_as_float(u);
}
__device__ __forceinline__ int float_to_ordered_int(float f) {
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float ordered_int_to_float(int i) {
  return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF);
}

__device__ __forceinline__ float sigmoidf_ref(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }


// One candidate: key = ~orderable(score) << 32 | (anchor * nc + class); slot claimed with an atomic per image.
__device__ __forceinline__ void emit_candidate(uint64_t* keys, int* img_count, long long cap_per_image, int img,
                                               int anchor_flat, int n_classes, int k, float score) {
  const int slot = atomicAdd(&img_count[img], 1);
  if (slot < cap_per_image)
    keys[static_cast<long long>(img) * cap_per_image + slot] =
        (static_cast<uint64_t>(orderable_desc(score)) << 32) | static_cast<uint32_t>(anchor_flat * n_classes + k);
}

// Box of one anchor in the reference's op order (yolort/models/_utils.py:59-60, torchvision box_convert).
__device__ __forceinline__ float4 decode_box(float sx, float sy, float sw, float sh, int x, int y, float stride_px,
                                             float aw, float ah) {
  const float cx = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sx, 2.0f), 0.5f), static_cast<float>(x)), stride_px);
  const float cy = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sy, 2.0f), 0.5f), static_cast<float>(y)), stride_px);
  const float tw = __fmul_rn(sw, 2.0f), th = __fmul_rn(sh, 2.0f);
  const float w = __fmul_rn(__fmul_rn(tw, tw), aw);
  const float h = __fmul_rn(__fmul_rn(th, th), ah);
  const float hw = __fmul_rn(0.5f, w), hh = __fmul_rn(0.5f, h);
  return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}

// The same box of a test-time-augmentation pass: (cx, cy, w, h) divided by the pass scale (IEEE fp32 division, as
// `p[..., :4] /= scale`, v5/models/yolo.py:181), cx = Wb - cx for the mirrored pass (:185), then the corner conversion.
__device__ __forceinline__ float4 decode_box_descaled(float sx, float sy, float sw, float sh, int x, int y, float stride_px,
                                                      float aw, float ah, float scale, bool flip, float flip_w) {
  float cx = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sx, 2.0f), 0.5f), static_cast<float>(x)), stride_px);
  float cy = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sy, 2.0f), 0.5f), static_cast<float>(y)), stride_px);
  const float tw = __fmul_rn(sw, 2.0f), th = __fmul_rn(sh, 2.0f);
  float w = __fmul_rn(__fmul_rn(tw, tw), aw);
  float h = __fmul_rn(__fmul_rn(th, th), ah);
  cx = __fdiv_rn(cx, scale);
  cy = __fdiv_rn(cy, scale);
  w = __fdiv_rn(w, scale);
  h = __fdiv_rn(h, scale);
  if (flip) cx = __fsub_rn(flip_w, cx);
  const float hw = __fmul_rn(0.5f, w), hh = __fmul_rn(0.5f, h);
  return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}

}  // namespace yb
