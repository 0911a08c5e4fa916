// Device code shared by the YOLOv5 augmentation kernels of v5_augment.cu: OpenCV 4.x's fixed-point bilinear remap
// (warpAffine / warpPerspective, border 114) over any source a tap functor describes, its BGR<->HSV conversions and the
// per-image LUT, and mixup's IEEE double blend.  oracle/restate_v5aug.py states each step.
#pragma once
#include "common.cuh"

namespace yb {
namespace v5 {

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

// OpenCV's fixed-point bilinear remap of output pixel (y, x) of an out_h x out_w warp with inverse map m: source taps
// at (sy + dy, sx + dx) with weights from the 5-bit fractions.  tap(ty, tx, p, stride_c) returns false for a tap that
// reads the border value, else points p at the tap's first channel.
template <class Tap>
__device__ __forceinline__ void warp_pixel(const double* m, bool perspective, int out_h, int out_w, int y, int x,
                                           const Tap& tap, uint32_t (&c)[3]) {
  const double yd = double(y);
  int X, Y;
  if (perspective) {
    // WarpPerspectiveInvoker sums each coordinate from its block's first column
    const int bw = min(1024 / min(16, out_h), out_w);
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
      const uint8_t* s;
      int64_t sc;
      if (tap(ty, tx, s, sc)) {
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] += int(__ldg(s + k * sc)) * wgt;
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

// Thread t's share of the HSV tables and the image's LUT, for the YB_V5_TO_HSV / YB_V5_LUT bits of `ops`
// (blockDim.x == 256; the caller synchronises).
__device__ __forceinline__ void load_colour_tables(Smem& sm, int ops, const uint8_t (&lut)[3][256], int t) {
  if (ops & YB_V5_TO_HSV) {
    // hsv_shift = 12 tables: saturate_cast<int>((255 << 12) / (1. * v)) and ((180 << 12) / (6. * diff))
    sm.sdiv[t] = t ? __double2int_rn(__ddiv_rn(double(255 << kHsvShift), double(t))) : 0;
    sm.hdiv[t] = t ? __double2int_rn(__ddiv_rn(double(180 << kHsvShift), __dmul_rn(6.0, double(t)))) : 0;
  }
  if (ops & YB_V5_LUT) {
#pragma unroll
    for (int k = 0; k < 3; ++k) sm.lut[k][t] = lut[k][t];
  }
}

// BGR->HSV, LUT, HSV->BGR, each when its bit is set, for the pixel at column x of a row of w before the flips.
// RGB2HSV / HSV2RGB are BGR2HSV / HSV2BGR with b and r swapped.
__device__ __forceinline__ void colour(uint32_t (&c)[3], int ops, const Smem& sm, int x, int w) {
  const bool rgb = ops & YB_V5_RGB;
  if (ops & YB_V5_TO_HSV) {
    if (rgb) swap_br(c);
    to_hsv(c, sm);
  }
  if (ops & YB_V5_LUT) {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = sm.lut[k][c[k]];
  }
  if (ops & YB_V5_FROM_HSV) {
    from_hsv(c, x, w);
    if (rgb) swap_br(c);
  }
}

// mixup: uint8(trunc(a * r + b * omr)) in IEEE double, omr = 1 - r as numpy computes it
__device__ __forceinline__ uint32_t mix(uint32_t a, uint32_t b, double r, double omr) {
  const double m = __dadd_rn(__dmul_rn(double(a), r), __dmul_rn(double(b), omr));
  return min(__double2uint_rz(m), 255u);
}

}  // namespace v5
}  // namespace yb
