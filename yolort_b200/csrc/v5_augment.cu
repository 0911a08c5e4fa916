// YOLOv5's own augmentations (yolort/v5/utils/augmentations.py: augment_hsv, random_perspective, cutout, mixup) on
// uint8 [H, W, 3] images, with OpenCV 4.x's arithmetic (oracle/restate_v5aug.py states it step by step).  Every
// random parameter was drawn on the host; an image's descriptor holds its inverse map, its 3 x 256 LUT, its flip and
// op bits and its cutout rectangles.
//
//   v5_augment_kernel   one launch for the batch: each output pixel maps back through the flips, then through the
//                       inverse warp (fixed-point source coordinates, 15-bit bilinear taps, border 114), then runs
//                       BGR->HSV (integer tables), the LUT (shared memory) and HSV->BGR (fp32), then the cutout
//                       rectangles; four consecutive pixels per thread, 12-byte stores along contiguous rows
//   v5_mixup_kernel     im * r + im2 * (1 - r) in IEEE double, truncated to uint8
//   v5_resize_kernel    load_image's cv2.resize(INTER_LINEAR) of the mosaic loader, OpenCV's 8-bit fixed point
//   v5_resize_area_kernel  load_image's cv2.resize(INTER_AREA) of the validation loader (augment=False)
//   v5_compose_kernel   one launch for a batch of training samples: the warp of each sample reads a virtual canvas
//                       (placed image views, 114 elsewhere), mixup, the colour steps and the flips, CHW stores
//                       (the two mosaic-loader kernels are restated in oracle/restate_v5mosaic.py)
//   v5_rescale_kernel   val.py's scale_coords / clip_coords of a batch's padded detections and its targets
//                       (INTER_AREA and the rescale are restated in oracle/restate_v5val.py)
//
// Built with -fmad=false (Makefile) and written with _rn intrinsics: every product and sum is rounded on its own, as
// OpenCV's x86 build rounds them; the two fused products of HSV2RGB are fmaf, as OpenCV's AVX2 build fuses them.
#include <cfloat>

#include "v5_augment.cuh"

namespace yb {
namespace {

using namespace v5;

// A tap of the image itself: outside it reads the border value.
struct ImageTap {
  const yb_v5_image& d;
  __device__ __forceinline__ bool operator()(int ty, int tx, const uint8_t*& s, int64_t& sc) const {
    if (ty >= 0 && ty < d.src_h && tx >= 0 && tx < d.src_w) {
      s = d.src + int64_t(ty) * d.src_stride_y + int64_t(tx) * d.src_stride_x;
      sc = d.src_stride_c;
      return true;
    }
    return false;
  }
};

__device__ __forceinline__ int find_image(const yb_v5_image* imgs, int n, int b) {
  int lo = 0, hi = n;                                   // first image with block_start > b
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (imgs[mid].block_start <= b) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

__global__ void __launch_bounds__(kThreads) v5_augment_kernel(const yb_v5_image* __restrict__ imgs, int n) {
  __shared__ Smem sm;
  const int b = int(blockIdx.x);
  const int i = find_image(imgs, n, b);
  const yb_v5_image& d = imgs[i];
  const int ops = d.ops;
  const int t = int(threadIdx.x);
  load_colour_tables(sm, ops, d.lut, t);
  __syncthreads();
  const int w = d.out_w;
  const int64_t plane = int64_t(d.out_h) * w;
  const int64_t p0 = int64_t(b - d.block_start) * kBlockPix + int64_t(t) * kPix;
  if (p0 >= plane) return;
  int y = int(p0 / w), x = int(p0 % w);
  uint8_t v[kPix][3];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (p0 + j < plane) {
      const int yf = (ops & YB_V5_FLIP_UD) ? d.out_h - 1 - y : y;
      const int xf = (ops & YB_V5_FLIP_LR) ? w - 1 - x : x;
      uint32_t c[3];
      if (ops & (YB_V5_AFFINE | YB_V5_PERSPECTIVE)) {
        warp_pixel(d.inv, ops & YB_V5_PERSPECTIVE, d.out_h, d.out_w, yf, xf, ImageTap{d}, c);
      } else {
        // no warp: the source is the output's shape, and may be the output itself (each pixel is read by the
        // thread that writes it, before it writes it)
        const uint8_t* s = d.src + int64_t(yf) * d.src_stride_y + int64_t(xf) * d.src_stride_x;
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = s[k * d.src_stride_c];
      }
      colour(c, ops, sm, xf, w);
      for (int r = 0; r < d.n_rects; ++r) {
        const int32_t* q = d.rects[r];
        if (y >= q[0] && x >= q[1] && y < q[2] && x < q[3]) {
          const uint32_t col = d.rect_color[r];
#pragma unroll
          for (int k = 0; k < 3; ++k) c[k] = (col >> (8 * k)) & 255u;
        }
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) v[j][k] = uint8_t(c[k]);
    }
    if (++x == w) {
      x = 0;
      ++y;
    }
  }
  const bool dense = d.dst_stride_c == 1 && d.dst_stride_x == 3 && d.dst_stride_y == 3 * int64_t(w);
  if (dense && p0 + kPix <= plane) {
    uint8_t* dst = d.dst + 3 * p0;
    if ((reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
      uint32_t word[3];
#pragma unroll
      for (int q = 0; q < 3; ++q)
        word[q] = uint32_t(v[(4 * q) / 3][(4 * q) % 3]) | (uint32_t(v[(4 * q + 1) / 3][(4 * q + 1) % 3]) << 8) |
                  (uint32_t(v[(4 * q + 2) / 3][(4 * q + 2) % 3]) << 16) |
                  (uint32_t(v[(4 * q + 3) / 3][(4 * q + 3) % 3]) << 24);
      *reinterpret_cast<uint3*>(dst) = make_uint3(word[0], word[1], word[2]);
      return;
    }
  }
  y = int(p0 / w);
  x = int(p0 % w);
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (p0 + j < plane) {
      uint8_t* o = d.dst + int64_t(y) * d.dst_stride_y + int64_t(x) * d.dst_stride_x;
#pragma unroll
      for (int k = 0; k < 3; ++k) o[k * d.dst_stride_c] = v[j][k];
    }
    if (++x == w) {
      x = 0;
      ++y;
    }
  }
}

__global__ void __launch_bounds__(kThreads) v5_mixup_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                                            uint8_t* __restrict__ dst, int64_t n, double r, double omr) {
  const int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= n) return;
  dst[i] = uint8_t(mix(a[i], b[i], r, omr));
}

// cv::resize's source position and 11-bit weights of output index d along an axis of ssz -> dsz: fx =
// float((d + 0.5) * scale - 0.5), s = floor(fx), weights saturate_cast<short>((1 - f) * 2048) and (f * 2048).  With
// `clamp` (the horizontal axis) a position outside [0, ssz - 1) takes the edge pixel with weights (2048, 0); the
// vertical axis keeps its weights and clamps the two rows it reads.
__device__ __forceinline__ void resize_coeffs(int d, int ssz, int dsz, bool clamp, int& s, int& w0, int& w1) {
  const double scale = __drcp_rn(__ddiv_rn(double(dsz), double(ssz)));
  float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn(double(d), 0.5), scale), 0.5));
  s = int(floorf(f));
  f = __fsub_rn(f, float(s));
  if (clamp && (s < 0 || s >= ssz - 1)) {
    s = s < 0 ? 0 : ssz - 1;
    f = 0.0f;
  }
  w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
  w1 = __float2int_rn(__fmul_rn(f, 2048.0f));
}

__device__ __forceinline__ int find_job(const yb_v5_resize_job* jobs, int n, int b) {
  int lo = 0, hi = n;                                   // first job with block_start > b
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (jobs[mid].block_start <= b) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

// INTER_AREA's taps of output index d along an axis of ssz -> dsz (computeResizeAreaTab, in IEEE double as the host
// computes them): a leading partial tap at s1 - 1, full taps s1 .. s2 - 1, a trailing partial tap at s2; each weight is
// rounded once to float.
struct AreaTaps {
  int s1, s2;
  bool lead, trail;
  float a_lead, a_full, a_trail;
};

__device__ __forceinline__ AreaTaps area_taps(int d, int ssz, double scale) {
  AreaTaps t;
  const double f1 = __dmul_rn(double(d), scale);
  const double f2 = __dadd_rn(f1, scale);
  const double cell = fmin(scale, __dsub_rn(double(ssz), f1));
  t.s2 = min(int(floor(f2)), ssz - 1);
  t.s1 = min(int(ceil(f1)), t.s2);
  const double lead = __dsub_rn(double(t.s1), f1), trail = __dsub_rn(f2, double(t.s2));
  t.lead = lead > 1e-3;
  t.trail = trail > 1e-3;
  t.a_lead = __double2float_rn(__ddiv_rn(lead, cell));
  t.a_full = __double2float_rn(__ddiv_rn(1.0, cell));
  t.a_trail = __double2float_rn(__ddiv_rn(fmin(fmin(trail, 1.0), cell), cell));
  return t;
}

__device__ __forceinline__ int area_tap(const AreaTaps& t, int k, float& a) {
  // tap k of 0 .. count-1 in table order
  if (t.lead) {
    if (k == 0) {
      a = t.a_lead;
      return t.s1 - 1;
    }
    --k;
  }
  if (k < t.s2 - t.s1) {
    a = t.a_full;
    return t.s1 + k;
  }
  a = t.a_trail;
  return t.s2;
}

__device__ __forceinline__ int area_count(const AreaTaps& t) { return int(t.lead) + (t.s2 - t.s1) + int(t.trail); }

// cv::resize(INTER_AREA) of one 8-bit output pixel, both axes shrinking.  Integer factors (both scales within
// DBL_EPSILON of an integer): 2 x 2 is (sum + 2) >> 2, any other ix x iy cvRound(float(sum) * (1.f / (ix * iy))).
// Otherwise ResizeArea_Invoker's order: per source row tap, buf = sum over the column taps of float(S) * alpha, in tap
// order; the output row's first row tap sets sum = beta * buf, each further one adds sum += beta * buf; cvRound(sum).
__device__ __forceinline__ void area_pixel(const yb_v5_resize_job& j, int dy, int dx, uint8_t* o) {
  const double scale_x = __drcp_rn(__ddiv_rn(double(j.dst_w), double(j.src_w)));
  const double scale_y = __drcp_rn(__ddiv_rn(double(j.dst_h), double(j.src_h)));
  const int ix = __double2int_rn(scale_x), iy = __double2int_rn(scale_y);
  const int64_t sy_ = j.src_stride_y, sx_ = j.src_stride_x, sc_ = j.src_stride_c;
  if (fabs(__dsub_rn(scale_x, double(ix))) < DBL_EPSILON && fabs(__dsub_rn(scale_y, double(iy))) < DBL_EPSILON) {
    const uint8_t* s = j.src + int64_t(dy) * iy * sy_ + int64_t(dx) * ix * sx_;
    const float inv = __fdiv_rn(1.0f, float(ix * iy));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      int sum = 0;
      for (int y = 0; y < iy; ++y)
        for (int x = 0; x < ix; ++x) sum += int(__ldg(s + y * sy_ + x * sx_ + k * sc_));
      o[k] = uint8_t(ix == 2 && iy == 2 ? (sum + 2) >> 2 : min(max(__float2int_rn(__fmul_rn(float(sum), inv)), 0), 255));
    }
    return;
  }
  const AreaTaps tx = area_taps(dx, j.src_w, scale_x), ty = area_taps(dy, j.src_h, scale_y);
  const int nx = area_count(tx), ny = area_count(ty);
  float sum[3] = {0.0f, 0.0f, 0.0f};
  for (int r = 0; r < ny; ++r) {
    float beta;
    const uint8_t* row = j.src + int64_t(area_tap(ty, r, beta)) * sy_;
    float buf[3] = {0.0f, 0.0f, 0.0f};
    for (int c = 0; c < nx; ++c) {
      float alpha;
      const uint8_t* s = row + int64_t(area_tap(tx, c, alpha)) * sx_;
#pragma unroll
      for (int k = 0; k < 3; ++k) buf[k] = __fadd_rn(buf[k], __fmul_rn(float(__ldg(s + k * sc_)), alpha));
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) sum[k] = r == 0 ? __fmul_rn(beta, buf[k]) : __fadd_rn(sum[k], __fmul_rn(beta, buf[k]));
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = uint8_t(min(max(__float2int_rn(sum[k]), 0), 255));
}

// One output pixel per thread.  INTER_LINEAR: the horizontal pass S = src[sx] * a0 + src[sx + 1] * a1 of rows sy and
// sy + 1, then ((S0 >> 4) * b0 >> 16) + ((S1 >> 4) * b1 >> 16) + 2 >> 2 (VResizeLinear's 8-bit form, vector and
// scalar alike).  An exact 2x downscale is INTER_AREA in OpenCV: (the 2 x 2 sum + 2) >> 2.
__global__ void __launch_bounds__(kThreads) v5_resize_kernel(const yb_v5_resize_job* __restrict__ jobs, int n) {
  const int b = int(blockIdx.x);
  const yb_v5_resize_job& j = jobs[find_job(jobs, n, b)];
  const int64_t p = int64_t(b - j.block_start) * kThreads + threadIdx.x;
  if (p >= int64_t(j.dst_h) * j.dst_w) return;
  const int dy = int(p / j.dst_w), dx = int(p % j.dst_w);
  uint8_t* o = j.dst + 3 * p;
  const uint8_t* src = j.src;
  const int64_t sy_ = j.src_stride_y, sx_ = j.src_stride_x, sc_ = j.src_stride_c;
  if (2 * j.dst_w == j.src_w && 2 * j.dst_h == j.src_h) {
    const uint8_t* s = src + int64_t(2 * dy) * sy_ + int64_t(2 * dx) * sx_;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const uint8_t* q = s + k * sc_;
      o[k] = uint8_t((int(__ldg(q)) + int(__ldg(q + sx_)) + int(__ldg(q + sy_)) + int(__ldg(q + sy_ + sx_)) + 2) >> 2);
    }
    return;
  }
  int sx, a0, a1, sy, b0, b1;
  resize_coeffs(dx, j.src_w, j.dst_w, true, sx, a0, a1);
  resize_coeffs(dy, j.src_h, j.dst_h, false, sy, b0, b1);
  const int sx1 = min(sx + 1, j.src_w - 1);
  const int r0 = min(max(sy, 0), j.src_h - 1), r1 = min(max(sy + 1, 0), j.src_h - 1);
  const uint8_t* p0 = src + int64_t(r0) * sy_;
  const uint8_t* p1 = src + int64_t(r1) * sy_;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int64_t c0 = int64_t(sx) * sx_ + k * sc_, c1 = int64_t(sx1) * sx_ + k * sc_;
    const int s0 = int(__ldg(p0 + c0)) * a0 + int(__ldg(p0 + c1)) * a1;
    const int s1 = int(__ldg(p1 + c0)) * a0 + int(__ldg(p1 + c1)) * a1;
    const int v = ((((s0 >> 4) * b0) >> 16) + (((s1 >> 4) * b1) >> 16) + 2) >> 2;
    o[k] = uint8_t(min(max(v, 0), 255));
  }
}

// cv2.resize(INTER_AREA), one output pixel per thread.  A kernel of its own: its double tap arithmetic would raise
// v5_resize_kernel's registers.
__global__ void __launch_bounds__(kThreads) v5_resize_area_kernel(const yb_v5_resize_job* __restrict__ jobs, int n) {
  const int b = int(blockIdx.x);
  const yb_v5_resize_job& j = jobs[find_job(jobs, n, b)];
  const int64_t p = int64_t(b - j.block_start) * kThreads + threadIdx.x;
  if (p >= int64_t(j.dst_h) * j.dst_w) return;
  area_pixel(j, int(p / j.dst_w), int(p % j.dst_w), j.dst + 3 * p);
}

// A tap of a virtual canvas: the placement holding it, or the border value 114.
struct CanvasTap {
  const yb_v5_canvas& cv;
  __device__ __forceinline__ bool operator()(int ty, int tx, const uint8_t*& s, int64_t& sc) const {
    for (int i = 0; i < cv.n_places; ++i) {
      const yb_v5_place& q = cv.places[i];
      if (ty >= q.y0 && ty < q.y1 && tx >= q.x0 && tx < q.x1) {
        s = q.src + int64_t(ty - q.oy) * q.stride_y + int64_t(tx - q.ox) * q.stride_x;
        sc = q.stride_c;
        return true;
      }
    }
    return false;
  }
};

__device__ __forceinline__ void canvas_pixel(const yb_v5_canvas& cv, int out_h, int out_w, int y, int x,
                                             uint32_t (&c)[3]) {
  if (cv.warp) {
    warp_pixel(cv.inv, cv.warp == YB_V5_PERSPECTIVE, out_h, out_w, y, x, CanvasTap{cv}, c);
    return;
  }
  const uint8_t* s;
  int64_t sc;
  if (CanvasTap{cv}(y, x, s, sc)) {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = __ldg(s + k * sc);
  } else {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = kBorder;
  }
}

// One launch for the batch: blockIdx.y is the sample, four consecutive pixels per thread; each pixel maps back
// through the flips, takes its canvases' warps (and mixup), runs the colour steps, and stores one byte per channel
// plane, four at a time along rows of planar output.
__global__ void __launch_bounds__(kThreads) v5_compose_kernel(const yb_v5_sample* __restrict__ samples) {
  __shared__ Smem sm;
  const yb_v5_sample& d = samples[blockIdx.y];
  const int ops = d.ops;
  const int t = int(threadIdx.x);
  load_colour_tables(sm, ops, d.lut, t);
  __syncthreads();
  const int w = d.out_w, h = d.out_h;
  const int64_t plane = int64_t(h) * w;
  const int64_t p0 = int64_t(blockIdx.x) * kBlockPix + int64_t(t) * kPix;
  if (p0 >= plane) return;
  int y = int(p0 / w), x = int(p0 % w);
  const int y_first = y, x_first = x;
  uint32_t v[kPix][3];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (p0 + j < plane) {
      const int yf = (ops & YB_V5_FLIP_UD) ? h - 1 - y : y;
      const int xf = (ops & YB_V5_FLIP_LR) ? w - 1 - x : x;
      uint32_t c[3];
      canvas_pixel(d.canvas[0], h, w, yf, xf, c);
      if (d.n_canvases == 2) {
        uint32_t c2[3];
        canvas_pixel(d.canvas[1], h, w, yf, xf, c2);
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = mix(c[k], c2[k], d.mix_r, d.mix_omr);
      }
      colour(c, ops, sm, xf, w);
#pragma unroll
      for (int k = 0; k < 3; ++k) v[j][k] = c[k];
    }
    if (++x == w) {
      x = 0;
      ++y;
    }
  }
  const bool rows4 = d.dst_stride_x == 1 && x_first + kPix <= w && p0 + kPix <= plane;
  uint8_t* o = d.dst + int64_t(y_first) * d.dst_stride_y + x_first;
  if (rows4 && ((reinterpret_cast<uintptr_t>(o) | uintptr_t(d.dst_stride_c)) & 3) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
      *reinterpret_cast<uint32_t*>(o + k * d.dst_stride_c) =
          v[0][k] | (v[1][k] << 8) | (v[2][k] << 16) | (v[3][k] << 24);
    return;
  }
  y = y_first;
  x = x_first;
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (p0 + j < plane) {
      uint8_t* q = d.dst + int64_t(y) * d.dst_stride_y + int64_t(x) * d.dst_stride_x;
#pragma unroll
      for (int k = 0; k < 3; ++k) q[k * d.dst_stride_c] = uint8_t(v[j][k]);
    }
    if (++x == w) {
      x = 0;
      ++y;
    }
  }
}

// scale_coords(img1_shape, coords, img0_shape, ratio_pad) then clip_coords in torch's CPU float32 arithmetic: x - pad,
// divided by gain with correct rounding (the python scalars rounded to float32), clamp to [0, w0] and [0, h0] with NaN
// passed through as torch.clamp passes it.  On CUDA tensors torch multiplies by the float reciprocal of gain instead,
// which can differ from this quotient by one unit in the last place.
__device__ __forceinline__ float clamp_torch(float v, float hi) {
  v = v < 0.0f ? 0.0f : v;
  return v > hi ? hi : v;
}

__device__ __forceinline__ void rescale_box(const float* prm, float (&b)[4]) {
  b[0] = clamp_torch(__fdiv_rn(__fsub_rn(b[0], prm[1]), prm[0]), prm[4]);
  b[1] = clamp_torch(__fdiv_rn(__fsub_rn(b[1], prm[2]), prm[0]), prm[3]);
  b[2] = clamp_torch(__fdiv_rn(__fsub_rn(b[2], prm[1]), prm[0]), prm[4]);
  b[3] = clamp_torch(__fdiv_rn(__fsub_rn(b[3], prm[2]), prm[0]), prm[3]);
}

// Threads [0, n * D) take the detections (slot d < counts[i] only); threads [n * D, n * D + T) the targets, which go
// first through val.py's targets[:, 2:] *= [W, H, W, H] and xywh2xyxy (w / 2 is w * 0.5 on the device).
__global__ void __launch_bounds__(kThreads) v5_rescale_kernel(yb_v5_rescale r) {
  const int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t nd = int64_t(r.n) * r.D;
  if (i < nd) {
    const int img = int(i / r.D);
    if (int(i % r.D) >= r.counts[img]) return;
    float4* p = reinterpret_cast<float4*>(r.boxes) + i;
    const float4 v = *p;
    float b[4] = {v.x, v.y, v.z, v.w};
    rescale_box(r.params + 5 * img, b);
    *p = make_float4(b[0], b[1], b[2], b[3]);
    return;
  }
  const int64_t t = i - nd;
  if (t >= r.T) return;
  const float* s = r.targets + 6 * t;
  float* o = r.targets_out + 6 * t;
  const float fi = s[0];
  o[0] = fi;
  o[1] = s[1];
  const float x = __fmul_rn(s[2], r.canvas_w), y = __fmul_rn(s[3], r.canvas_h);
  const float hw = __fmul_rn(__fmul_rn(s[4], r.canvas_w), 0.5f), hh = __fmul_rn(__fmul_rn(s[5], r.canvas_h), 0.5f);
  float b[4] = {__fsub_rn(x, hw), __fsub_rn(y, hh), __fadd_rn(x, hw), __fadd_rn(y, hh)};
  const int img = int(fi);
  if (fi == float(img) && img >= 0 && img < r.n) rescale_box(r.params + 5 * img, b);
#pragma unroll
  for (int k = 0; k < 4; ++k) o[2 + k] = b[k];
}

int64_t blocks_for(int64_t pixels) { return (pixels + kBlockPix - 1) / kBlockPix; }

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_v5_augment_prepare(int n_images, yb_v5_image* images, int64_t* total_blocks) {
  YB_REQUIRE(n_images > 0 && images && total_blocks, "v5_augment_prepare: null argument or empty batch");
  int64_t blocks = 0;
  for (int i = 0; i < n_images; ++i) {
    yb_v5_image& d = images[i];
    YB_REQUIRE(d.src && d.dst && d.src_h > 0 && d.src_w > 0 && d.out_h > 0 && d.out_w > 0,
               "v5_augment_prepare: image %d has no pixels", i);
    YB_REQUIRE(d.out_h < (1 << 24) && d.out_w < (1 << 24), "v5_augment_prepare: image %d: output beyond 2^24 a side",
               i);
    const int warp = d.ops & (YB_V5_AFFINE | YB_V5_PERSPECTIVE);
    YB_REQUIRE(warp != (YB_V5_AFFINE | YB_V5_PERSPECTIVE), "v5_augment_prepare: image %d: affine and perspective", i);
    YB_REQUIRE(warp || (d.src_h == d.out_h && d.src_w == d.out_w),
               "v5_augment_prepare: image %d: without a warp the output is the source's size", i);
    YB_REQUIRE(d.src != d.dst || !(d.ops & (YB_V5_AFFINE | YB_V5_PERSPECTIVE | YB_V5_FLIP_LR | YB_V5_FLIP_UD)),
               "v5_augment_prepare: image %d: in place only without warp and flips", i);
    YB_REQUIRE(d.n_rects >= 0 && d.n_rects <= YB_V5_MAX_RECTS, "v5_augment_prepare: image %d has %d rectangles", i,
               d.n_rects);
    d.block_start = int32_t(blocks);
    blocks += blocks_for(int64_t(d.out_h) * d.out_w);
    YB_REQUIRE(blocks < (int64_t(1) << 31), "v5_augment_prepare: batch too large");
  }
  *total_blocks = blocks;
  return YB_OK;
}

extern "C" int yb_v5_augment(int n_images, const yb_v5_image* images_dev, int64_t total_blocks, void* stream_) {
  YB_REQUIRE(n_images > 0 && images_dev && total_blocks > 0, "v5_augment: null argument or empty batch");
  v5_augment_kernel<<<unsigned(total_blocks), kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(images_dev,
                                                                                                 n_images);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_v5_mixup(const uint8_t* a_dev, const uint8_t* b_dev, uint8_t* dst_dev, int64_t n, double r,
                           void* stream_) {
  YB_REQUIRE(a_dev && b_dev && dst_dev && n > 0, "v5_mixup: null argument or no pixels");
  const int64_t blocks = (n + kThreads - 1) / kThreads;
  YB_REQUIRE(blocks < (int64_t(1) << 31), "v5_mixup: image too large");
  // 1 - r as numpy computes it: one double subtraction on the host
  v5_mixup_kernel<<<unsigned(blocks), kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(a_dev, b_dev, dst_dev, n, r,
                                                                                         1.0 - r);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

namespace yb {
namespace {
int resize_prepare(const char* what, bool area, int n_jobs, yb_v5_resize_job* jobs, int64_t* total_blocks) {
  YB_REQUIRE(n_jobs > 0 && jobs && total_blocks, "%s: null argument or no jobs", what);
  int64_t blocks = 0;
  for (int i = 0; i < n_jobs; ++i) {
    yb_v5_resize_job& j = jobs[i];
    YB_REQUIRE(j.src && j.dst && j.src_h > 0 && j.src_w > 0 && j.dst_h > 0 && j.dst_w > 0, "%s: job %d has no pixels",
               what, i);
    YB_REQUIRE(j.src_h < (1 << 24) && j.src_w < (1 << 24) && j.dst_h < (1 << 24) && j.dst_w < (1 << 24),
               "%s: job %d: beyond 2^24 a side", what, i);
    YB_REQUIRE(!area || (j.dst_h <= j.src_h && j.dst_w <= j.src_w), "%s: job %d: %d x %d -> %d x %d does not shrink",
               what, i, j.src_h, j.src_w, j.dst_h, j.dst_w);
    j.block_start = int32_t(blocks);
    blocks += (int64_t(j.dst_h) * j.dst_w + kThreads - 1) / kThreads;
    YB_REQUIRE(blocks < (int64_t(1) << 31), "%s: batch too large", what);
  }
  *total_blocks = blocks;
  return YB_OK;
}
}  // namespace
}  // namespace yb

extern "C" int yb_v5_resize_prepare(int n_jobs, yb_v5_resize_job* jobs, int64_t* total_blocks) {
  return resize_prepare("v5_resize_prepare", false, n_jobs, jobs, total_blocks);
}

extern "C" int yb_v5_resize(int n_jobs, const yb_v5_resize_job* jobs_dev, int64_t total_blocks, void* stream_) {
  YB_REQUIRE(n_jobs > 0 && jobs_dev && total_blocks > 0, "v5_resize: null argument or no jobs");
  v5_resize_kernel<<<unsigned(total_blocks), kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(jobs_dev, n_jobs);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_v5_resize_area_prepare(int n_jobs, yb_v5_resize_job* jobs, int64_t* total_blocks) {
  return resize_prepare("v5_resize_area_prepare", true, n_jobs, jobs, total_blocks);
}

extern "C" int yb_v5_resize_area(int n_jobs, const yb_v5_resize_job* jobs_dev, int64_t total_blocks, void* stream_) {
  YB_REQUIRE(n_jobs > 0 && jobs_dev && total_blocks > 0, "v5_resize_area: null argument or no jobs");
  v5_resize_area_kernel<<<unsigned(total_blocks), kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(jobs_dev,
                                                                                                    n_jobs);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_v5_compose_prepare(int n_samples, const yb_v5_sample* samples, int64_t* blocks_per_sample) {
  YB_REQUIRE(n_samples > 0 && n_samples < 65536 && samples && blocks_per_sample,
             "v5_compose_prepare: null argument, or not 1..65535 samples");
  const int oh = samples[0].out_h, ow = samples[0].out_w;
  YB_REQUIRE(oh > 0 && ow > 0 && oh < (1 << 24) && ow < (1 << 24), "v5_compose_prepare: output of %d x %d", oh, ow);
  for (int i = 0; i < n_samples; ++i) {
    const yb_v5_sample& d = samples[i];
    YB_REQUIRE(d.dst && d.out_h == oh && d.out_w == ow, "v5_compose_prepare: sample %d: no output, or not %d x %d",
               i, oh, ow);
    YB_REQUIRE(d.n_canvases == 1 || d.n_canvases == 2, "v5_compose_prepare: sample %d has %d canvases", i,
               d.n_canvases);
    YB_REQUIRE(!(d.ops & (YB_V5_AFFINE | YB_V5_PERSPECTIVE)), "v5_compose_prepare: sample %d: warps are per canvas", i);
    for (int c = 0; c < d.n_canvases; ++c) {
      const yb_v5_canvas& cv = d.canvas[c];
      YB_REQUIRE(cv.warp == 0 || cv.warp == YB_V5_AFFINE || cv.warp == YB_V5_PERSPECTIVE,
                 "v5_compose_prepare: sample %d canvas %d: warp %d", i, c, cv.warp);
      YB_REQUIRE(cv.n_places >= 0 && cv.n_places <= YB_V5_MAX_PLACES,
                 "v5_compose_prepare: sample %d canvas %d has %d placements", i, c, cv.n_places);
      for (int p = 0; p < cv.n_places; ++p)
        YB_REQUIRE(cv.places[p].src, "v5_compose_prepare: sample %d canvas %d placement %d has no source", i, c, p);
    }
  }
  *blocks_per_sample = blocks_for(int64_t(oh) * ow);
  YB_REQUIRE(*blocks_per_sample < (int64_t(1) << 31), "v5_compose_prepare: output too large");
  return YB_OK;
}

extern "C" int yb_v5_compose(int n_samples, const yb_v5_sample* samples_dev, int64_t blocks_per_sample,
                             void* stream_) {
  YB_REQUIRE(n_samples > 0 && n_samples < 65536 && samples_dev && blocks_per_sample > 0,
             "v5_compose: null argument or no samples");
  const dim3 grid{unsigned(blocks_per_sample), unsigned(n_samples), 1u};
  v5_compose_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(samples_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_v5_rescale_coords(const yb_v5_rescale* r, void* stream_) {
  YB_REQUIRE(r && r->n >= 0 && r->D >= 0 && r->T >= 0, "v5_rescale_coords: null argument or negative size");
  const int64_t nd = int64_t(r->n) * r->D;
  YB_REQUIRE(nd == 0 || (r->boxes && r->counts && (reinterpret_cast<uintptr_t>(r->boxes) & 15) == 0),
             "v5_rescale_coords: boxes and counts are required (boxes 16-byte aligned)");
  YB_REQUIRE(r->T == 0 || (r->targets && r->targets_out), "v5_rescale_coords: targets need an output");
  YB_REQUIRE(r->params || (nd == 0 && r->T == 0), "v5_rescale_coords: no params");
  const int64_t blocks = (nd + r->T + kThreads - 1) / kThreads;
  if (blocks == 0) return YB_OK;
  YB_REQUIRE(blocks < (int64_t(1) << 31), "v5_rescale_coords: too many boxes");
  v5_rescale_kernel<<<unsigned(blocks), kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(*r);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
