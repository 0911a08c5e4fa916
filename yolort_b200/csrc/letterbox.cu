// Letterbox pre-processing: aspect-preserving bilinear resize + centred pad, whole batch in one launch.
//
// Replaces YOLOTransform.forward (yolort/models/transform.py:143-221):
//   _resize_image_and_masks :53-97  -> F.interpolate(bilinear, align_corners=False,
//                                      recompute_scale_factor=True), i.e. ATen upsample_bilinear2d
//   batch_images            :297-330 -> new_full(fill) + centred copy
// and fuses the uint8 -> [0,1] conversion of the default loader (yolov5.py:218-228) plus the layout
// change the first convolution wants (space-to-depth NHWC, see conv_sm90.cu / engine.py).
//
// HBM-bound: per image it reads 3*h*w source bytes and writes the canvas once.  The hot variant
// (letterbox_s2d_tile_kernel: uint8 sources -> the plan's space-to-depth canvas) stages the source rectangle of a
// 16 x 128 pixel output tile in shared memory with 16-byte coalesced loads and samples from there, so every source
// byte crosses the memory system once as part of a full 16-byte request; the generic kernels below sample global
// memory directly (consecutive threads -> consecutive output x, source texels reused through L1/L2).
#include <cmath>
#include <type_traits>

#include "common.cuh"

namespace yb {
namespace {

constexpr int kMaxImagesPerLaunch = 64;
constexpr int kRowsPerBlock = 8;   // s2d rows per CTA (amortises the 1 KB LUT staging)

struct ImgGeom {
  const void* src;
  int src_h, src_w, new_h, new_w, top, left;
  float ratio_h, ratio_w;
};
// Element strides (channel, row, pixel) of the source: planar CHW = (h*w, w, 1); interleaved HWC (what image
// decoders emit) = (1, 3w, 3).  A template parameter, so the planar path keeps its constant-stride addressing.
template <bool kHwc>
struct SrcStrides {
  size_t cs, rs, ps;
  __device__ __forceinline__ explicit SrcStrides(const ImgGeom& g)
      : cs(kHwc ? 1 : static_cast<size_t>(g.src_h) * g.src_w), rs(kHwc ? 3 * static_cast<size_t>(g.src_w) : g.src_w),
        ps(kHwc ? 3 : 1) {}
};
struct BatchGeom {
  ImgGeom img[kMaxImagesPerLaunch];
};

template <typename SrcT>
__device__ __forceinline__ float load_src(const SrcT* p, const float* lut);
template <>
__device__ __forceinline__ float load_src<uint8_t>(const uint8_t* p, const float* lut) {
  return lut[__ldg(p)];   // `lut` points to the shared-memory copy staged by the kernel
}
template <>
__device__ __forceinline__ float load_src<float>(const float* p, const float*) {
  return __ldg(p);
}
template <>
__device__ __forceinline__ float load_src<__half>(const __half* p, const float*) {
  return __half2float(__ldg(p));
}
template <>
__device__ __forceinline__ float load_src<__nv_bfloat16>(const __nv_bfloat16* p, const float*) {
  return __bfloat162float(*p);
}

// Source index / interpolation weight exactly as ATen's area_pixel_compute_source_index +
// guard_index_and_lambda (align_corners=False, no antialias), all in fp32.
__device__ __forceinline__ void src_coord(int dst, float ratio, int size, int& i0, int& i1, float& l1) {
  float real = __fsub_rn(__fmul_rn(ratio, static_cast<float>(dst) + 0.5f), 0.5f);
  if (real < 0.f) real = 0.f;
  int idx = static_cast<int>(real);
  if (idx > size - 1) idx = size - 1;
  float lam = __fsub_rn(real, static_cast<float>(idx));
  lam = fminf(fmaxf(lam, 0.f), 1.f);
  i0 = idx;
  i1 = idx + (idx < size - 1 ? 1 : 0);
  l1 = lam;
}

template <typename SrcT, bool kHwc>
__device__ __forceinline__ void sample_rgb(const ImgGeom& g, const float* lut, int y, int x, float fill,
                                           float (&rgb)[3]) {
  const int yy = y - g.top, xx = x - g.left;
  if (yy < 0 || yy >= g.new_h || xx < 0 || xx >= g.new_w) {
    rgb[0] = rgb[1] = rgb[2] = fill;
    return;
  }
  const SrcStrides<kHwc> st(g);
  if (g.new_h == g.src_h && g.new_w == g.src_w) {
    // identity resize (ratios are exactly 1, all interpolation weights exactly 0/1): plain copy, same bits
    const SrcT* base = static_cast<const SrcT*>(g.src);
    const size_t o = static_cast<size_t>(yy) * st.rs + static_cast<size_t>(xx) * st.ps;
#pragma unroll
    for (int c = 0; c < 3; ++c) rgb[c] = load_src<SrcT>(base + static_cast<size_t>(c) * st.cs + o, lut);
    return;
  }
  int y0, y1, x0, x1;
  float ly, lx;
  src_coord(yy, g.ratio_h, g.src_h, y0, y1, ly);
  src_coord(xx, g.ratio_w, g.src_w, x0, x1, lx);
  const float wy0 = 1.f - ly, wx0 = 1.f - lx;
  const SrcT* base = static_cast<const SrcT*>(g.src);
  const size_t r0 = static_cast<size_t>(y0) * st.rs, r1 = static_cast<size_t>(y1) * st.rs;
  const size_t c0 = static_cast<size_t>(x0) * st.ps, c1 = static_cast<size_t>(x1) * st.ps;
  // Taps with zero weight are not fetched (w*p + 0*q == w*p exactly for finite q): an identity resize
  // (the 640x640 headline case) touches one source texel per output pixel instead of four.
  const bool need_x1 = lx != 0.f, need_y1 = ly != 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const SrcT* p = base + static_cast<size_t>(c) * st.cs;
    const float p00 = load_src<SrcT>(p + r0 + c0, lut);
    const float p01 = need_x1 ? load_src<SrcT>(p + r0 + c1, lut) : p00;
    float bot = 0.f;
    if (need_y1) {
      const float p10 = load_src<SrcT>(p + r1 + c0, lut);
      const float p11 = need_x1 ? load_src<SrcT>(p + r1 + c1, lut) : p10;
      bot = __fadd_rn(__fmul_rn(wx0, p10), __fmul_rn(lx, p11));
    }
    const float top = __fadd_rn(__fmul_rn(wx0, p00), __fmul_rn(lx, p01));
    rgb[c] = __fadd_rn(__fmul_rn(wy0, top), __fmul_rn(ly, bot));
  }
}

template <typename DstT>
__device__ __forceinline__ DstT cvt_out(float v);
template <>
__device__ __forceinline__ float cvt_out<float>(float v) {
  return v;
}
template <>
__device__ __forceinline__ __half cvt_out<__half>(float v) {
  return __float2half_rn(v);
}
template <>
__device__ __forceinline__ __nv_bfloat16 cvt_out<__nv_bfloat16>(float v) {
  return __float2bfloat16_rn(v);
}

// byte -> float without a conversion instruction: 0x4B000000 | b is the float 2^23 + b, exactly; subtracting 2^23 leaves b.
// (The conversion pipe, I2F / F2F, runs at a fraction of the ALU rate: the uint8 -> fp16 canvas was bound by it, ~48 us
// for 39 M values whatever the memory access pattern.)
__device__ __forceinline__ float byte_to_float(uint32_t word, int k) {   // byte k (0..3) of `word`
  return __fsub_rn(__uint_as_float(__byte_perm(word, 0x4B000000u, 0x7540u | static_cast<uint32_t>(k))), 8388608.0f);
}
// two floats -> two 16-bit values with ONE packed conversion instruction
template <typename DstT>
__device__ __forceinline__ uint32_t cvt_pack2(float a, float b);
template <>
__device__ __forceinline__ uint32_t cvt_pack2<__half>(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
template <>
__device__ __forceinline__ uint32_t cvt_pack2<__nv_bfloat16>(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// NCHW destination (reference layout): thread per (y, x), three planes.
template <typename SrcT, typename DstT, bool kHwc>
__global__ void letterbox_nchw_kernel(const __grid_constant__ BatchGeom bg, int img0, int Hb, int Wb,
                                      float fill, const float* lut, DstT* __restrict__ dst) {
  __shared__ float s_lut[256];
  if (lut != nullptr) {   // uint8 sources: one coalesced 1 KB read per CTA instead of a global lookup per texel
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = lut[i];
    __syncthreads();
    lut = s_lut;
  }
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int li = blockIdx.z;
  if (x >= Wb) return;
  float rgb[3];
  sample_rgb<SrcT, kHwc>(bg.img[li], lut, y, x, fill, rgb);
  const size_t plane = static_cast<size_t>(Hb) * Wb;
  DstT* o = dst + static_cast<size_t>(img0 + li) * 3 * plane + static_cast<size_t>(y) * Wb + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * plane] = cvt_out<DstT>(rgb[c]);
}

// Space-to-depth NHWC destination [N, Hb/2, Wb/2, 16]: thread per 2x2 pixel block, one 32-byte store.
template <typename SrcT, typename DstT, bool kHwc>
__global__ void letterbox_s2d_kernel(const __grid_constant__ BatchGeom bg, int img0, int Hb, int Wb,
                                     float fill, const float* lut, DstT* __restrict__ dst) {
  __shared__ float s_lut[256];
  if (lut != nullptr) {   // uint8 sources: one coalesced 1 KB read per CTA instead of a global lookup per texel
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = lut[i];
    __syncthreads();
    lut = s_lut;
  }
  const int X = blockIdx.x * blockDim.x + threadIdx.x;
  const int li = blockIdx.z;
  const int W2 = Wb >> 1, H2 = Hb >> 1;
  if (X >= W2) return;
  for (int Y = blockIdx.y * kRowsPerBlock; Y < min(H2, (blockIdx.y + 1) * kRowsPerBlock); ++Y) {
    __align__(16) DstT v[16];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        float rgb[3];
        sample_rgb<SrcT, kHwc>(bg.img[li], lut, 2 * Y + dy, 2 * X + dx, fill, rgb);
        const int q = (dy * 2 + dx) * 4;
        v[q + 0] = cvt_out<DstT>(rgb[0]);
        v[q + 1] = cvt_out<DstT>(rgb[1]);
        v[q + 2] = cvt_out<DstT>(rgb[2]);
        v[q + 3] = cvt_out<DstT>(0.f);
      }
    }
    DstT* o = dst + ((static_cast<size_t>(img0 + li) * H2 + Y) * W2 + X) * 16;
    reinterpret_cast<uint4*>(o)[0] = reinterpret_cast<const uint4*>(v)[0];
    reinterpret_cast<uint4*>(o)[1] = reinterpret_cast<const uint4*>(v)[1];
  }
}

// ---- tiled variant: uint8 sources -> space-to-depth canvas, source rectangle staged in shared memory -----------------
constexpr int kTileY = 8, kTileX = 64;            // s2d pixels per CTA tile: 16 x 128 canvas pixels
constexpr int kTileThreads = 256;
constexpr int kTileSmem = 40 * 1024;              // staging bytes (covers down-scaling ratios up to ~2.2, e.g. 1280 -> 640)
constexpr int kTileMaxLines = 3 * 40;

// Same arithmetic as sample_rgb, texels read from the staged rectangle: `line(c, y)` / `col(c, x)` address it.
template <bool kHwc>
struct StagedSrc {
  const uint8_t* buf;
  const uint16_t* mis;      // per line: misalignment of the line start inside its first 16-byte chunk
  int pitch, rows, y_lo, x_lo;
  __device__ __forceinline__ float at(const float* lut, int c, int y, int x) const {
    const int line = kHwc ? (y - y_lo) : c * rows + (y - y_lo);
    const int byte = kHwc ? 3 * (x - x_lo) + c : (x - x_lo);
    return lut[buf[line * pitch + mis[line] + byte]];
  }
};

template <bool kHwc>
__device__ __forceinline__ void sample_rgb_staged(const ImgGeom& g, const StagedSrc<kHwc>& S, const float* lut, int y, int x,
                                                  float fill, float (&rgb)[3]) {
  const int yy = y - g.top, xx = x - g.left;
  if (yy < 0 || yy >= g.new_h || xx < 0 || xx >= g.new_w) {
    rgb[0] = rgb[1] = rgb[2] = fill;
    return;
  }
  if (g.new_h == g.src_h && g.new_w == g.src_w) {
#pragma unroll
    for (int c = 0; c < 3; ++c) rgb[c] = S.at(lut, c, yy, xx);
    return;
  }
  int y0, y1, x0, x1;
  float ly, lx;
  src_coord(yy, g.ratio_h, g.src_h, y0, y1, ly);
  src_coord(xx, g.ratio_w, g.src_w, x0, x1, lx);
  const float wy0 = 1.f - ly, wx0 = 1.f - lx;
  const bool need_x1 = lx != 0.f, need_y1 = ly != 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float p00 = S.at(lut, c, y0, x0);
    const float p01 = need_x1 ? S.at(lut, c, y0, x1) : p00;
    float bot = 0.f;
    if (need_y1) {
      const float p10 = S.at(lut, c, y1, x0);
      const float p11 = need_x1 ? S.at(lut, c, y1, x1) : p10;
      bot = __fadd_rn(__fmul_rn(wx0, p10), __fmul_rn(lx, p11));
    }
    const float top = __fadd_rn(__fmul_rn(wx0, p00), __fmul_rn(lx, p01));
    rgb[c] = __fadd_rn(__fmul_rn(wy0, top), __fmul_rn(ly, bot));
  }
}

template <typename DstT, bool kHwc>
__global__ void __launch_bounds__(kTileThreads)
letterbox_s2d_tile_kernel(const __grid_constant__ BatchGeom bg, int img0, int Hb, int Wb, float fill, const float* lut,
                          DstT* __restrict__ dst, int smem_bytes) {
  __shared__ float s_lut[256];
  extern __shared__ __align__(16) uint8_t s_src[];   // staging bytes: `smem_bytes` (sized by the host for this batch)
  __shared__ uint16_t s_mis[kTileMaxLines];
  __shared__ int s_rect[7];   // y_lo, rows, x_lo, cols, pitch, staged?, identity tile fully inside the image?
  const int tid = threadIdx.x;
  const int li = blockIdx.z;
  const ImgGeom& g = bg.img[li];
  const int W2 = Wb >> 1, H2 = Hb >> 1;
  const int X0 = blockIdx.x * kTileX, Y0 = blockIdx.y * kTileY;
  s_lut[tid] = lut[tid];
  // canvas rows / columns of this tile that fall inside the resized image
  const int cy0 = max(2 * Y0, g.top), cy1 = min(min(2 * (Y0 + kTileY), Hb), g.top + g.new_h) - 1;
  const int cx0 = max(2 * X0, g.left), cx1 = min(min(2 * (X0 + kTileX), Wb), g.left + g.new_w) - 1;
  const bool any = cy0 <= cy1 && cx0 <= cx1;
  if (tid == 0) {
    int y_lo = 0, y_hi = -1, x_lo = 0, x_hi = -1;
    if (any) {
      if (g.new_h == g.src_h && g.new_w == g.src_w) {
        y_lo = cy0 - g.top; y_hi = cy1 - g.top; x_lo = cx0 - g.left; x_hi = cx1 - g.left;
      } else {
        int a, b;
        float l;
        src_coord(cy0 - g.top, g.ratio_h, g.src_h, y_lo, b, l);
        src_coord(cy1 - g.top, g.ratio_h, g.src_h, a, y_hi, l);
        src_coord(cx0 - g.left, g.ratio_w, g.src_w, x_lo, b, l);
        src_coord(cx1 - g.left, g.ratio_w, g.src_w, a, x_hi, l);
      }
    }
    const int rows = y_hi - y_lo + 1, cols = x_hi - x_lo + 1;
    const int line_bytes = kHwc ? 3 * cols : cols;
    const int pitch = (line_bytes + 15 + 15) / 16 * 16;     // room for the leading misalignment
    const int lines = kHwc ? rows : 3 * rows;
    s_rect[0] = y_lo; s_rect[1] = rows; s_rect[2] = x_lo; s_rect[3] = cols; s_rect[4] = pitch;
    s_rect[5] = (any && lines <= kTileMaxLines && lines * pitch <= smem_bytes) ? 1 : 0;
    // identity resize and every canvas pixel of the tile inside the image: the copy fast path below (no per-pixel
    // bounds / interpolation logic; the 640 x 640 headline case is all such tiles)
    s_rect[6] = (s_rect[5] && g.new_h == g.src_h && g.new_w == g.src_w && cy0 == 2 * Y0 && cx0 == 2 * X0 &&
                 cy1 == 2 * (Y0 + kTileY) - 1 && cx1 == 2 * (X0 + kTileX) - 1) ? 1 : 0;
  }
  __syncthreads();
  const int y_lo = s_rect[0], rows = s_rect[1], x_lo = s_rect[2], cols = s_rect[3], pitch = s_rect[4];
  const bool staged = s_rect[5] != 0;
  const uint8_t* base = static_cast<const uint8_t*>(g.src);
  if (staged) {
    const int lines = kHwc ? rows : 3 * rows;
    const int line_bytes = kHwc ? 3 * cols : cols;
    const int cpl = pitch >> 4;                                // 16-byte chunks per staged line
    const size_t plane = static_cast<size_t>(g.src_h) * g.src_w;
    for (int idx = tid; idx < lines * cpl; idx += kTileThreads) {
      const int line = idx / cpl, ch = idx - line * cpl;
      const int c = kHwc ? 0 : line / rows, r = kHwc ? line : line - c * rows;
      const size_t off = kHwc ? (static_cast<size_t>(y_lo + r) * g.src_w + x_lo) * 3
                              : static_cast<size_t>(c) * plane + static_cast<size_t>(y_lo + r) * g.src_w + x_lo;
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(base + off);
      const uintptr_t al = a0 & ~static_cast<uintptr_t>(15);
      if (ch == 0) s_mis[line] = static_cast<uint16_t>(a0 - al);
      const uintptr_t p = al + static_cast<uintptr_t>(ch) * 16;
      // an aligned 16-byte chunk that holds at least one byte of the line lies inside the mapped page of that byte
      if (p < a0 + line_bytes)
        *reinterpret_cast<uint4*>(&s_src[line * pitch + ch * 16]) = __ldg(reinterpret_cast<const uint4*>(p));
    }
  }
  __syncthreads();
  StagedSrc<kHwc> S{s_src, s_mis, pitch, rows, y_lo, x_lo};
  // Work item = HALF a space-to-depth pixel: canvas row 2Y + dy, columns 2X and 2X + 1, i.e. 16 contiguous output
  // bytes.  Consecutive lanes take consecutive halves, so a warp's store instruction writes one contiguous 512-byte
  // run (4 lines); with a whole pixel per thread the 16-byte pieces sat 32 bytes apart (8 lines per instruction) and the
  // store wavefronts, not DRAM, bounded the kernel (see letterbox_s2d_identity_kernel below).
  constexpr int kHalves = 2 * kTileY * kTileX;                      // 1024 per tile
  const bool copy = s_rect[6] != 0;
#pragma unroll
  for (int k = 0; k < kHalves / kTileThreads; ++k) {
    const int hp = tid + k * kTileThreads;
    const int dy = hp & 1, xs = (hp >> 1) & (kTileX - 1), Yl = hp / (2 * kTileX);
    const int X = X0 + xs, Y = Y0 + Yl;
    if (X >= W2 || Y >= H2) continue;
    float f[2][3];
    if (copy) {
      // copy fast path (identity resize, tile fully inside the image): the two horizontally adjacent bytes of a
      // (row, channel) sit side by side in the staged line; bytes become floats without a conversion instruction and
      // half(byte * (1/255)) equals half(torch's byte / 255.0) for all 256 byte values (tests/test_host_logic.py)
      const int r = 2 * Yl + dy, bx = 2 * xs;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int line = kHwc ? r : c * rows + r;
        const uint8_t* ln = s_src + line * pitch + s_mis[line] + (kHwc ? 3 * bx + c : bx);
        f[0][c] = __fmul_rn(byte_to_float(ln[0], 0), 1.0f / 255.0f);
        f[1][c] = __fmul_rn(byte_to_float(ln[kHwc ? 3 : 1], 0), 1.0f / 255.0f);
      }
    } else {
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        if (staged)
          sample_rgb_staged<kHwc>(g, S, s_lut, 2 * Y + dy, 2 * X + dx, fill, f[dx]);
        else if (any)
          sample_rgb<uint8_t, kHwc>(g, s_lut, 2 * Y + dy, 2 * X + dx, fill, f[dx]);
        else
          f[dx][0] = f[dx][1] = f[dx][2] = fill;
      }
    }
    uint8_t* o = reinterpret_cast<uint8_t*>(dst + ((static_cast<size_t>(img0 + li) * H2 + Y) * W2 + X) * 16) + dy * 16;
    *reinterpret_cast<uint4*>(o) = make_uint4(cvt_pack2<DstT>(f[0][0], f[0][1]), cvt_pack2<DstT>(f[0][2], 0.f),
                                              cvt_pack2<DstT>(f[1][0], f[1][1]), cvt_pack2<DstT>(f[1][2], 0.f));
  }
}

// Identity resize of planar uint8 images that cover the whole canvas (pre-sized inputs: the 640 x 640 headline case and
// any serving front end that resizes on the host): nothing to interpolate, nothing to pad.  What bounds this copy is
// the number of 128-byte lines a STORE instruction touches (one L1 wavefront per line), not arithmetic: with a thread
// per space-to-depth pixel a warp's 16-byte stores sit 32 bytes apart (8 lines per instruction, the tile kernel's copy
// path), with a thread per 8 canvas pixels 128 bytes apart (32 lines).  Here LANE l WRITES
// BYTES [16 l, 16 l + 16) of a 512-byte run: lane (x, dy) = (l / 2, l % 2) converts canvas row 2Y + dy, columns 2X,
// 2X + 1 (three 2-byte loads; even / odd lanes read two source rows, 32 contiguous bytes each) into its half of
// space-to-depth pixel X -- four lines per store instruction, four such runs per warp.
// byte * (1/255) in fp32 then ONE packed conversion per value pair; half(byte * (1/255)) equals half(torch's byte / 255.0)
// for all 256 byte values (tests/test_host_logic.py).
constexpr int kIdRuns = 4;      // 512-byte runs (16 space-to-depth pixels each) per warp
template <typename DstT>
__global__ void __launch_bounds__(256)
letterbox_s2d_identity_kernel(const __grid_constant__ BatchGeom bg, int img0, int Hb, int Wb, DstT* __restrict__ dst) {
  const int li = blockIdx.z;
  const int H2 = Hb >> 1, W2 = Wb >> 1;
  const int xblocks = (W2 + 16 * kIdRuns - 1) / (16 * kIdRuns);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= xblocks * H2) return;
  const int Y = warp / xblocks, xb = warp - Y * xblocks;
  const int dy = lane & 1, xo = lane >> 1;
  const uint8_t* base = static_cast<const uint8_t*>(bg.img[li].src) + static_cast<size_t>(2 * Y + dy) * Wb;
  const size_t plane = static_cast<size_t>(Hb) * Wb;
  uint16_t in[kIdRuns][3];
#pragma unroll
  for (int r = 0; r < kIdRuns; ++r) {
    const int X = xb * 16 * kIdRuns + r * 16 + xo;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      in[r][c] = X < W2 ? __ldg(reinterpret_cast<const uint16_t*>(base + c * plane + 2 * X)) : static_cast<uint16_t>(0);
  }
  uint8_t* orow = reinterpret_cast<uint8_t*>(dst + (static_cast<size_t>(img0 + li) * H2 + Y) * W2 * 16);
#pragma unroll
  for (int r = 0; r < kIdRuns; ++r) {
    const int X = xb * 16 * kIdRuns + r * 16 + xo;
    float f[2][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      f[0][c] = __fmul_rn(byte_to_float(in[r][c], 0), 1.0f / 255.0f);
      f[1][c] = __fmul_rn(byte_to_float(in[r][c], 1), 1.0f / 255.0f);
    }
    if (X < W2)
      *reinterpret_cast<uint4*>(orow + static_cast<size_t>(X) * 32 + dy * 16) =
          make_uint4(cvt_pack2<DstT>(f[0][0], f[0][1]), cvt_pack2<DstT>(f[0][2], 0.f), cvt_pack2<DstT>(f[1][0], f[1][1]),
                     cvt_pack2<DstT>(f[1][2], 0.f));
  }
}

template <typename SrcT, typename DstT, bool kHwc>
int launch_typed(const BatchGeom& bg, int img0, int count, int Hb, int Wb, float fill, const float* lut,
                 void* dst, int layout, cudaStream_t stream) {
  const int threads = 128;
  if (layout == YB_LAYOUT_NCHW) {
    dim3 grid((Wb + threads - 1) / threads, Hb, count);
    letterbox_nchw_kernel<SrcT, DstT, kHwc><<<grid, threads, 0, stream>>>(bg, img0, Hb, Wb, fill, lut,
                                                                    static_cast<DstT*>(dst));
  } else if constexpr (std::is_same<SrcT, uint8_t>::value && sizeof(DstT) == 2) {
    if constexpr (!kHwc) {
      bool identity = (Wb % 2 == 0) && (Hb % 2 == 0);
      for (int j = 0; j < count && identity; ++j) {
        const ImgGeom& g = bg.img[j];
        identity = g.src_h == Hb && g.src_w == Wb && g.new_h == Hb && g.new_w == Wb && g.top == 0 && g.left == 0 &&
                   (reinterpret_cast<uintptr_t>(g.src) & 1) == 0;
      }
      if (identity) {
        const int warps_total = ((Wb / 2 + 16 * kIdRuns - 1) / (16 * kIdRuns)) * (Hb / 2);
        dim3 grid((warps_total * 32 + 255) / 256, 1, count);
        letterbox_s2d_identity_kernel<DstT><<<grid, 256, 0, stream>>>(bg, img0, Hb, Wb, static_cast<DstT*>(dst));
        YB_CHECK_CUDA(cudaGetLastError());
        return YB_OK;
      }
    }
    dim3 grid((Wb / 2 + kTileX - 1) / kTileX, (Hb / 2 + kTileY - 1) / kTileY, count);
    // staging bytes for the largest source rectangle of a 16 x 128 output tile in this batch (identity resizes need
    // 8 KB, a 2x down-scale ~31 KB): small footprints let more CTAs share an SM and hide the load -> sample latency
    int need = 0;
    for (int j = 0; j < count; ++j) {
      const ImgGeom& g = bg.img[j];
      const int rows = static_cast<int>(2 * kTileY * g.ratio_h) + 3, cols = static_cast<int>(2 * kTileX * g.ratio_w) + 3;
      const int line_bytes = kHwc ? 3 * cols : cols;
      const int bytes = (kHwc ? rows : 3 * rows) * ((line_bytes + 30) / 16 * 16);
      if (bytes > need) need = bytes;
    }
    if (need > kTileSmem) need = kTileSmem;       // larger rectangles take the direct-sampling path inside the kernel
    need = (need + 1023) / 1024 * 1024;
    letterbox_s2d_tile_kernel<DstT, kHwc><<<grid, kTileThreads, need, stream>>>(bg, img0, Hb, Wb, fill, lut, static_cast<DstT*>(dst), need);
  } else {
    dim3 grid((Wb / 2 + threads - 1) / threads, (Hb / 2 + kRowsPerBlock - 1) / kRowsPerBlock, count);
    letterbox_s2d_kernel<SrcT, DstT, kHwc><<<grid, threads, 0, stream>>>(bg, img0, Hb, Wb, fill, lut,
                                                                   static_cast<DstT*>(dst));
  }
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

template <typename SrcT, bool kHwc>
int launch_src(const BatchGeom& bg, int img0, int count, int Hb, int Wb, float fill, const float* lut,
               void* dst, int dst_dtype, int layout, cudaStream_t stream) {
  switch (dst_dtype) {
    case YB_F32:
      if (layout == YB_LAYOUT_S2D16) break;
      return launch_typed<SrcT, float, kHwc>(bg, img0, count, Hb, Wb, fill, lut, dst, layout, stream);
    case YB_F16:
      return launch_typed<SrcT, __half, kHwc>(bg, img0, count, Hb, Wb, fill, lut, dst, layout, stream);
    case YB_BF16:
      return launch_typed<SrcT, __nv_bfloat16, kHwc>(bg, img0, count, Hb, Wb, fill, lut, dst, layout, stream);
    default:
      break;
  }
  set_error("letterbox: unsupported destination dtype %d for layout %d", dst_dtype, layout);
  return YB_ERR_INVALID;
}

// ---- test-time augmentation: rescaled (and mirrored) copies of a space-to-depth canvas --------------------------------
// scale_img (yolort/v5/utils/torch_utils.py:288-300) of `x.flip(3) if flip else x` (v5/models/yolo.py:157):
// F.interpolate(size=(nh, nw), bilinear, align_corners=False) then F.pad(right/bottom, 0.447).  The sample indices are
// src_coord's, computed in the mirrored frame; a mirrored tap at column i reads column Wb-1-i of the canvas.  Work item
// = half a space-to-depth pixel (canvas row 2Y+dy, columns 2X and 2X+1): 16 contiguous output bytes, consecutive
// threads -> consecutive items, so a warp stores one contiguous 512-byte run.  Each tap is one 8-byte load (the four
// channels of a pixel sit together in the source layout).  HBM-bound: the source canvas is read about once (neighbouring
// items share taps through L1/L2) and the pass canvas written once.
template <typename DstT>
__device__ __forceinline__ void load_px4(const DstT* img, int W2, int y, int x, float (&v)[3]) {
  const uint2 raw = __ldg(reinterpret_cast<const uint2*>(img + ((static_cast<size_t>(y >> 1) * W2 + (x >> 1)) * 16 +
                                                                ((y & 1) * 2 + (x & 1)) * 4)));
  const DstT* e = reinterpret_cast<const DstT*>(&raw);
  v[0] = static_cast<float>(e[0]);
  v[1] = static_cast<float>(e[1]);
  v[2] = static_cast<float>(e[2]);
}

template <typename DstT>
__global__ void __launch_bounds__(256)
canvas_rescale_kernel(const DstT* __restrict__ src, int Hb, int Wb, DstT* __restrict__ dst, int Hp, int Wp, int nh, int nw,
                      float ratio_h, float ratio_w, int flip, float fill, long long items_per_image, long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int n = static_cast<int>(i / items_per_image);
  const long long r = i - n * items_per_image;
  const int W2p = Wp >> 1;
  const int dy = static_cast<int>(r & 1);
  const int X = static_cast<int>((r >> 1) % W2p), Y = static_cast<int>((r >> 1) / W2p);
  const int y = 2 * Y + dy;
  const DstT* img = src + static_cast<size_t>(n) * (Hb >> 1) * (Wb >> 1) * 16;
  float f[2][3];
  int y0 = 0, y1 = 0;
  float ly = 0.f;
  if (y < nh) src_coord(y, ratio_h, Hb, y0, y1, ly);
  const float wy0 = 1.f - ly;
#pragma unroll
  for (int dx = 0; dx < 2; ++dx) {
    const int x = 2 * X + dx;
    if (y >= nh || x >= nw) {
      f[dx][0] = f[dx][1] = f[dx][2] = fill;
      continue;
    }
    int x0, x1;
    float lx;
    src_coord(x, ratio_w, Wb, x0, x1, lx);
    if (flip) {
      x0 = Wb - 1 - x0;
      x1 = Wb - 1 - x1;
    }
    const float wx0 = 1.f - lx;
    float p00[3], p01[3], p10[3], p11[3];
    load_px4<DstT>(img, Wb >> 1, y0, x0, p00);
    load_px4<DstT>(img, Wb >> 1, y0, x1, p01);
    load_px4<DstT>(img, Wb >> 1, y1, x0, p10);
    load_px4<DstT>(img, Wb >> 1, y1, x1, p11);
#pragma unroll
    for (int c = 0; c < 3; ++c) {   // sample_rgb's arithmetic: fp32, unfused, one rounding at the store
      const float top = __fadd_rn(__fmul_rn(wx0, p00[c]), __fmul_rn(lx, p01[c]));
      const float bot = __fadd_rn(__fmul_rn(wx0, p10[c]), __fmul_rn(lx, p11[c]));
      f[dx][c] = __fadd_rn(__fmul_rn(wy0, top), __fmul_rn(ly, bot));
    }
  }
  uint8_t* o = reinterpret_cast<uint8_t*>(dst + static_cast<size_t>(n) * (Hp >> 1) * W2p * 16) + r * 16;
  *reinterpret_cast<uint4*>(o) = make_uint4(cvt_pack2<DstT>(f[0][0], f[0][1]), cvt_pack2<DstT>(f[0][2], 0.f),
                                            cvt_pack2<DstT>(f[1][0], f[1][1]), cvt_pack2<DstT>(f[1][2], 0.f));
}

}  // namespace
}  // namespace yb

extern "C" int yb_canvas_rescale(int n, const void* src_dev, int dtype, int Hb, int Wb, int nh, int nw, int flip_lr,
                                 float fill, void* dst_dev, int Hp, int Wp, void* stream_) {
  using namespace yb;
  YB_REQUIRE(n > 0 && src_dev && dst_dev, "canvas_rescale: null/empty arguments");
  YB_REQUIRE(dtype == YB_F16 || dtype == YB_BF16, "canvas_rescale: canvas dtype must be fp16 or bf16");
  YB_REQUIRE(Hb > 0 && Wb > 0 && Hp > 0 && Wp > 0 && Hb % 2 == 0 && Wb % 2 == 0 && Hp % 2 == 0 && Wp % 2 == 0,
             "canvas_rescale: canvases must have positive, even sizes");
  YB_REQUIRE(nh > 0 && nw > 0 && nh <= Hp && nw <= Wp, "canvas_rescale: resized area %dx%d does not fit %dx%d", nh, nw,
             Hp, Wp);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(src_dev) & 7) == 0 && (reinterpret_cast<uintptr_t>(dst_dev) & 15) == 0,
             "canvas_rescale: misaligned canvas");
  // upsample_bilinear2d with an output size and no scale factor: ratio = float(in) / out (area_pixel_compute_scale)
  const float ratio_h = static_cast<float>(Hb) / static_cast<float>(nh);
  const float ratio_w = static_cast<float>(Wb) / static_cast<float>(nw);
  const long long items = static_cast<long long>(Hp / 2) * (Wp / 2) * 2;
  const long long total = items * n;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (dtype == YB_F16)
    canvas_rescale_kernel<__half><<<blocks, 256, 0, stream>>>(static_cast<const __half*>(src_dev), Hb, Wb,
                                                              static_cast<__half*>(dst_dev), Hp, Wp, nh, nw, ratio_h,
                                                              ratio_w, flip_lr ? 1 : 0, fill, items, total);
  else
    canvas_rescale_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(src_dev), Hb, Wb, static_cast<__nv_bfloat16*>(dst_dev), Hp, Wp, nh, nw, ratio_h,
        ratio_w, flip_lr ? 1 : 0, fill, items, total);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_letterbox_geometry(int n, const int32_t* src_hw, float min_size, float max_size,
                                     int size_divisible, const int32_t* fixed_shape,
                                     yb_letterbox_geom* geom, int32_t* batch_hw) {
  YB_REQUIRE(n > 0 && src_hw && geom && batch_hw, "letterbox_geometry: null/empty arguments");
  YB_REQUIRE(size_divisible > 0, "letterbox_geometry: size_divisible must be positive");
  int max_h = 0, max_w = 0;
  for (int i = 0; i < n; ++i) {
    const int h = src_hw[2 * i], w = src_hw[2 * i + 1];
    YB_REQUIRE(h > 0 && w > 0, "letterbox_geometry: image %d has non-positive size", i);
    const int lo = h < w ? h : w, hi = h < w ? w : h;
    // transform.py:66-73: python-float / fp32 0-dim tensor == tensor.reciprocal() * scalar, in fp32.
    volatile float ra = 1.0f / static_cast<float>(lo);
    volatile float rb = 1.0f / static_cast<float>(hi);
    volatile float a = ra * min_size;
    volatile float b = rb * max_size;
    const double s = static_cast<double>(a < b ? a : b);
    const int nh = static_cast<int>(static_cast<double>(h) * s);
    const int nw = static_cast<int>(static_cast<double>(w) * s);
    YB_REQUIRE(nh > 0 && nw > 0, "letterbox_geometry: image %d resizes to an empty image", i);
    geom[i].src_h = h;
    geom[i].src_w = w;
    geom[i].new_h = nh;
    geom[i].new_w = nw;
    geom[i].ratio_h = static_cast<float>(h) / static_cast<float>(nh);
    geom[i].ratio_w = static_cast<float>(w) / static_cast<float>(nw);
    if (nh > max_h) max_h = nh;
    if (nw > max_w) max_w = nw;
  }
  int Hb, Wb;
  if (fixed_shape) {
    Hb = fixed_shape[0];
    Wb = fixed_shape[1];
    YB_REQUIRE(Hb >= max_h && Wb >= max_w, "letterbox_geometry: fixed_shape (%d,%d) smaller than resized (%d,%d)",
               Hb, Wb, max_h, max_w);
  } else {
    const double d = static_cast<double>(size_divisible);
    Hb = static_cast<int>(std::ceil(static_cast<double>(max_h) / d) * d);
    Wb = static_cast<int>(std::ceil(static_cast<double>(max_w) / d) * d);
  }
  for (int i = 0; i < n; ++i) {
    // transform.py:322-326: int(round(d/2 - 0.1)), Python round == round-half-even on doubles.
    geom[i].top = static_cast<int>(std::nearbyint((Hb - geom[i].new_h) / 2.0 - 0.1));
    geom[i].left = static_cast<int>(std::nearbyint((Wb - geom[i].new_w) / 2.0 - 0.1));
  }
  batch_hw[0] = Hb;
  batch_hw[1] = Wb;
  return YB_OK;
}

extern "C" int yb_scale_coords_params(int Hb, int Wb, int src_h, int src_w, float* out3) {
  YB_REQUIRE(out3 && src_h > 0 && src_w > 0, "scale_coords_params: bad arguments");
  // transform.py:358-359 on fp32 tensors: gain = min(Hb/h, Wb/w); pad = (Wb - w*gain)/2, (Hb - h*gain)/2
  volatile float gh = static_cast<float>(Hb) / static_cast<float>(src_h);
  volatile float gw = static_cast<float>(Wb) / static_cast<float>(src_w);
  volatile float gain = gh < gw ? gh : gw;
  volatile float wx = static_cast<float>(src_w) * gain;
  volatile float hy = static_cast<float>(src_h) * gain;
  volatile float px = (static_cast<float>(Wb) - wx) / 2.0f;
  volatile float py = (static_cast<float>(Hb) - hy) / 2.0f;
  out3[0] = gain;
  out3[1] = px;
  out3[2] = py;
  return YB_OK;
}

extern "C" int yb_letterbox(int n, const void* const* src_dev, int src_dtype, const yb_letterbox_geom* geom,
                            int Hb, int Wb, float fill, const float* u8_lut_dev, void* dst_dev,
                            int dst_dtype, int dst_layout, void* stream_) {
  return yb_letterbox_strided(n, src_dev, src_dtype, YB_SRC_CHW, geom, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype,
                              dst_layout, stream_);
}

extern "C" int yb_letterbox_strided(int n, const void* const* src_dev, int src_dtype, int src_layout,
                                    const yb_letterbox_geom* geom, int Hb, int Wb, float fill,
                                    const float* u8_lut_dev, void* dst_dev, int dst_dtype, int dst_layout,
                                    void* stream_) {
  using namespace yb;
  YB_REQUIRE(src_layout == YB_SRC_CHW || src_layout == YB_SRC_HWC, "letterbox: bad source layout %d", src_layout);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(n > 0 && src_dev && geom && dst_dev, "letterbox: null/empty arguments");
  YB_REQUIRE(dst_layout == YB_LAYOUT_NCHW || dst_layout == YB_LAYOUT_S2D16, "letterbox: bad layout");
  YB_REQUIRE(dst_layout != YB_LAYOUT_S2D16 || (Hb % 2 == 0 && Wb % 2 == 0),
             "letterbox: S2D16 layout needs even canvas size");
  YB_REQUIRE(src_dtype != YB_U8 || u8_lut_dev != nullptr, "letterbox: uint8 sources need the 256-entry LUT");
  for (int i0 = 0; i0 < n; i0 += kMaxImagesPerLaunch) {
    const int count = (n - i0) < kMaxImagesPerLaunch ? (n - i0) : kMaxImagesPerLaunch;
    BatchGeom bg;
    for (int j = 0; j < count; ++j) {
      const yb_letterbox_geom& g = geom[i0 + j];
      YB_REQUIRE(g.top >= 0 && g.left >= 0 && g.top + g.new_h <= Hb && g.left + g.new_w <= Wb,
                 "letterbox: image %d does not fit the canvas", i0 + j);
      YB_REQUIRE(static_cast<long long>(g.src_h) * g.src_w * 3 < (1ll << 31), "letterbox: image %d too large", i0 + j);
      bg.img[j] = ImgGeom{src_dev[i0 + j], g.src_h, g.src_w, g.new_h, g.new_w, g.top, g.left, g.ratio_h, g.ratio_w};
    }
    int rc;
    const bool hwc = src_layout == YB_SRC_HWC;
    switch (src_dtype) {
      case YB_U8:
        rc = hwc ? launch_src<uint8_t, true>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream)
                 : launch_src<uint8_t, false>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream);
        break;
      case YB_F32:
        rc = hwc ? launch_src<float, true>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream)
                 : launch_src<float, false>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream);
        break;
      case YB_F16:
        rc = hwc ? launch_src<__half, true>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream)
                 : launch_src<__half, false>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream);
        break;
      case YB_BF16:
        rc = hwc ? launch_src<__nv_bfloat16, true>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream)
                 : launch_src<__nv_bfloat16, false>(bg, i0, count, Hb, Wb, fill, u8_lut_dev, dst_dev, dst_dtype, dst_layout, stream);
        break;
      default:
        set_error("letterbox: unsupported source dtype %d", src_dtype);
        return YB_ERR_INVALID;
    }
    if (rc != YB_OK) return rc;
  }
  return YB_OK;
}
