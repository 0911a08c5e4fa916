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
//
// Built with -fmad=false (Makefile) and written with _rn intrinsics: every product and sum is rounded on its own, as
// OpenCV's x86 build rounds them; the two fused products of HSV2RGB are fmaf, as OpenCV's AVX2 build fuses them.
#include "common.cuh"

namespace yb {
namespace {

constexpr int kThreads = 256;
constexpr int kPix = 4;                               // pixels per thread
constexpr int kBlockPix = kThreads * kPix;
constexpr int kHsvShift = 12;
constexpr int kHsvVec = 32;                           // HSV2RGB_b's vector step: 4 x v_float32 of 8 lanes (AVX2)
constexpr int kBorder = 114;

struct Smem {
  int sdiv[256];
  int hdiv[256];
  uint8_t lut[3][256];
};

// OpenCV's fixed-point bilinear remap of output pixel (y, x): source taps at (sy + dy, sx + dx) with weights from
// the 5-bit fractions; a tap outside the image reads the border value.
__device__ __forceinline__ void warp_pixel(const yb_v5_image& d, int y, int x, uint32_t (&c)[3]) {
  const double* m = d.inv;
  const double yd = double(y);
  int X, Y;
  if (d.ops & YB_V5_PERSPECTIVE) {
    // WarpPerspectiveInvoker sums each coordinate from its block's first column
    const int bw = min(1024 / min(16, d.out_h), d.out_w);
    const int xb = (x / bw) * bw;
    const double xbd = double(xb), x1 = double(x - xb);
    const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(m[0], xbd), __dmul_rn(m[1], yd)), m[2]);
    const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(m[3], xbd), __dmul_rn(m[4], yd)), m[5]);
    const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(m[6], xbd), __dmul_rn(m[7], yd)), m[8]);
    double W = __dadd_rn(W0, __dmul_rn(m[6], x1));
    W = W != 0.0 ? __ddiv_rn(32.0, W) : 0.0;
    const double lo = -2147483648.0, hi = 2147483647.0;
    const double fX = fmax(lo, fmin(hi, __dmul_rn(__dadd_rn(X0, __dmul_rn(m[0], x1)), W)));
    const double fY = fmax(lo, fmin(hi, __dmul_rn(__dadd_rn(Y0, __dmul_rn(m[3], x1)), W)));
    X = __double2int_rn(fX);
    Y = __double2int_rn(fY);
  } else {
    // warpAffine: AB_BITS = 10, round_delta = AB_SCALE / INTER_TAB_SIZE / 2 = 16
    const double xd = double(x);
    const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(m[0], xd), 1024.0));
    const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(m[3], xd), 1024.0));
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], yd), m[2]), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], yd), m[5]), 1024.0)) + 16;
    X = (X0 + adelta) >> 5;
    Y = (Y0 + bdelta) >> 5;
  }
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  const int ax = X & 31, ay = Y & 31;
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int wgt = ((dy ? ay : 32 - ay) * (dx ? ax : 32 - ax)) << 5;
      const int ty = sy + dy, tx = sx + dx;
      if (ty >= 0 && ty < d.src_h && tx >= 0 && tx < d.src_w) {
        const uint8_t* s = d.src + int64_t(ty) * d.src_stride_y + int64_t(tx) * d.src_stride_x;
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] += int(__ldg(s + k * d.src_stride_c)) * wgt;
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] += kBorder * wgt;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) c[k] = uint32_t((acc[k] + (1 << 14)) >> 15);
}

// COLOR_BGR2HSV (RGB2HSV_b): c = (b, g, r) in, (h, s, v) out.
__device__ __forceinline__ void to_hsv(uint32_t (&c)[3], const Smem& sm) {
  const int b = int(c[0]), g = int(c[1]), r = int(c[2]);
  const int v = max(max(b, g), r);
  const int diff = v - min(min(b, g), r);
  const int s = (diff * sm.sdiv[v] + (1 << (kHsvShift - 1))) >> kHsvShift;
  int h = v == r ? g - b : v == g ? b - r + 2 * diff : r - g + 4 * diff;
  h = (h * sm.hdiv[diff] + (1 << (kHsvShift - 1))) >> kHsvShift;
  h += h < 0 ? 180 : 0;
  c[0] = uint32_t(h);
  c[1] = uint32_t(s);
  c[2] = uint32_t(v);
}

// COLOR_HSV2BGR (HSV2RGB_b): c = (h, s, v) in, (b, g, r) out.  Pixel `x` of a row of `w`: the first
// floor(w / 32) * 32 of each row take OpenCV's vector path (sector by truncation, products truncated), the rest its
// scalar path (fmod / floor sector, products rounded to nearest even).
__device__ __forceinline__ void from_hsv(uint32_t (&c)[3], int x, int w) {
  const bool vec = x < (w / kHsvVec) * kHsvVec;
  const float h = __fmul_rn(__uint2float_rn(c[0]), 6.0f / 180.0f);
  const float s = __fmul_rn(__uint2float_rn(c[1]), 1.0f / 255.0f);
  const float v = __fmul_rn(__uint2float_rn(c[2]), 1.0f / 255.0f);
  int sector;
  float f;
  if (vec) {
    const float pre = truncf(h);
    f = __fsub_rn(h, pre);
    sector = int(__fsub_rn(pre, __fmul_rn(truncf(__fmul_rn(pre, 1.0f / 6.0f)), 6.0f)));
  } else {
    const float hs = fmodf(h, 6.0f);
    sector = int(floorf(hs));
    f = __fsub_rn(hs, float(sector));
    if (unsigned(sector) >= 6u) {
      sector = 0;
      f = 0.0f;
    }
  }
  const float tab1 = __fmul_rn(v, __fsub_rn(1.0f, s));
  const float tab2 = __fmul_rn(v, __fmaf_rn(-s, f, 1.0f));
  const float tab3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.0f, f), 1.0f));
  // sector_data {1,3,0}, {1,0,2}, {3,0,1}, {0,2,1}, {0,1,3}, {2,1,0}: the tab entries (b, g, r) take, 2 bits each
  constexpr uint64_t kSectors = 0x0Dull | 0x21ull << 6 | 0x13ull << 12 | 0x18ull << 18 | 0x34ull << 24 | 0x06ull << 30;
  const uint32_t sel = uint32_t(kSectors >> (6 * sector)) & 0x3Fu;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint32_t e = (sel >> (2 * k)) & 3u;
    const float o = __fmul_rn(e == 0 ? v : e == 1 ? tab1 : e == 2 ? tab2 : tab3, 255.0f);
    const int q = vec ? __float2int_rz(o) : __float2int_rn(o);
    c[k] = uint32_t(min(max(q, 0), 255));
  }
}

__device__ __forceinline__ void swap_br(uint32_t (&c)[3]) {
  const uint32_t t = c[0];
  c[0] = c[2];
  c[2] = t;
}

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
  if (ops & YB_V5_TO_HSV) {
    // hsv_shift = 12 tables: saturate_cast<int>((255 << 12) / (1. * v)) and ((180 << 12) / (6. * diff))
    sm.sdiv[t] = t ? __double2int_rn(__ddiv_rn(double(255 << kHsvShift), double(t))) : 0;
    sm.hdiv[t] = t ? __double2int_rn(__ddiv_rn(double(180 << kHsvShift), __dmul_rn(6.0, double(t)))) : 0;
  }
  if (ops & YB_V5_LUT) {
#pragma unroll
    for (int k = 0; k < 3; ++k) sm.lut[k][t] = d.lut[k][t];
  }
  __syncthreads();
  const int w = d.out_w;
  const int64_t plane = int64_t(d.out_h) * w;
  const int64_t p0 = int64_t(b - d.block_start) * kBlockPix + int64_t(t) * kPix;
  if (p0 >= plane) return;
  const bool rgb = ops & YB_V5_RGB;
  int y = int(p0 / w), x = int(p0 % w);
  uint8_t v[kPix][3];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (p0 + j < plane) {
      const int yf = (ops & YB_V5_FLIP_UD) ? d.out_h - 1 - y : y;
      const int xf = (ops & YB_V5_FLIP_LR) ? w - 1 - x : x;
      uint32_t c[3];
      if (ops & (YB_V5_AFFINE | YB_V5_PERSPECTIVE)) {
        warp_pixel(d, yf, xf, c);
      } else {
        // no warp: the source is the output's shape, and may be the output itself (each pixel is read by the
        // thread that writes it, before it writes it)
        const uint8_t* s = d.src + int64_t(yf) * d.src_stride_y + int64_t(xf) * d.src_stride_x;
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = s[k * d.src_stride_c];
      }
      // RGB2HSV / HSV2RGB are BGR2HSV / HSV2BGR with b and r swapped
      if (ops & YB_V5_TO_HSV) {
        if (rgb) swap_br(c);
        to_hsv(c, sm);
      }
      if (ops & YB_V5_LUT) {
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = sm.lut[k][c[k]];
      }
      if (ops & YB_V5_FROM_HSV) {
        from_hsv(c, xf, w);
        if (rgb) swap_br(c);
      }
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
  const double m = __dadd_rn(__dmul_rn(double(a[i]), r), __dmul_rn(double(b[i]), omr));
  dst[i] = uint8_t(min(__double2uint_rz(m), 255u));
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
