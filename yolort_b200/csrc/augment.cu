// Training augmentations on uint8 images: the reference's default_train_transforms on tensors, with torchvision's
// tensor arithmetic (oracle/restate_augment.py states it rule by rule).  Every random parameter was drawn on the host;
// an image's recipe is its list of ops in call order.
//
//   mean     one launch per contrast round: each pixel of the image the contrast op sees is rebuilt (mapped back
//            through the geometric ops before it, then the colour ops before it), its truncated grayscale value is
//            summed as an exact integer (block sums, one 64-bit integer atomicAdd per block: the total does not
//            depend on the order)
//   output   each output pixel is mapped back through flip, crop and zoom-out to a source pixel or a fill value,
//            then the colour chain runs on the RGB triple; four pixels per thread, 4-byte / 16-byte stores along
//            the rows of each plane where the plane's alignment allows
//
// Built with -fmad=false (Makefile) and written with _rn intrinsics: every product and sum is rounded on its own, as
// torch's CPU kernels round them.
#include "common.cuh"

namespace yb {
namespace {

constexpr int kThreads = 256;
constexpr int kPix = 4;                               // pixels per thread
constexpr int kBlockPix = kThreads * kPix;

struct Rgb {
  uint32_t c[3];
};

__device__ __forceinline__ uint32_t to_u8(float v) {   // clamp(0, 255) then .to(uint8): truncation
  return __float2uint_rz(fminf(fmaxf(v, 0.0f), 255.0f));
}

__device__ __forceinline__ uint32_t gray(const Rgb& p) {
  const float s = __fadd_rn(__fadd_rn(__fmul_rn(float(0.2989), __uint2float_rn(p.c[0])),
                                      __fmul_rn(float(0.587), __uint2float_rn(p.c[1]))),
                            __fmul_rn(float(0.114), __uint2float_rn(p.c[2])));
  return __float2uint_rz(s);
}

__device__ __forceinline__ uint32_t blend(uint32_t x, float other, float r, float omr) {
  return to_u8(__fadd_rn(__fmul_rn(r, __uint2float_rn(x)), __fmul_rn(omr, other)));
}

__device__ __forceinline__ void hue(Rgb& p, float factor) {
  const float r = __fdiv_rn(__uint2float_rn(p.c[0]), 255.0f);
  const float g = __fdiv_rn(__uint2float_rn(p.c[1]), 255.0f);
  const float b = __fdiv_rn(__uint2float_rn(p.c[2]), 255.0f);
  const float maxc = fmaxf(fmaxf(r, g), b), minc = fminf(fminf(r, g), b);
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.0f : maxc);
  const float crd = eqc ? 1.0f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd);
  const float gc = __fdiv_rn(__fsub_rn(maxc, g), crd);
  const float bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
  float h;
  if (maxc == r) h = __fsub_rn(bc, gc);
  else if (maxc == g) h = __fsub_rn(__fadd_rn(2.0f, rc), bc);
  else h = __fsub_rn(__fadd_rn(4.0f, gc), rc);
  h = fmodf(__fadd_rn(__fdiv_rn(h, 6.0f), 1.0f), 1.0f);
  h = fmodf(__fadd_rn(h, factor), 1.0f);              // torch.remainder(x, 1.0): fmod, plus 1 when negative
  if (h < 0.0f) h = __fadd_rn(h, 1.0f);
  const float h6 = __fmul_rn(h, 6.0f);
  const float fi = floorf(h6);
  const float f = __fsub_rn(h6, fi);
  const int i = int(fi) % 6;
  const float v = maxc;
  const float pp = fminf(fmaxf(__fmul_rn(v, __fsub_rn(1.0f, s)), 0.0f), 1.0f);
  const float q = fminf(fmaxf(__fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(s, f))), 0.0f), 1.0f);
  const float t = fminf(fmaxf(__fmul_rn(v, __fsub_rn(1.0f, __fmul_rn(s, __fsub_rn(1.0f, f)))), 0.0f), 1.0f);
  float o0, o1, o2;
  switch (i) {
    case 0: o0 = v; o1 = t; o2 = pp; break;
    case 1: o0 = q; o1 = v; o2 = pp; break;
    case 2: o0 = pp; o1 = v; o2 = t; break;
    case 3: o0 = pp; o1 = q; o2 = v; break;
    case 4: o0 = t; o1 = pp; o2 = v; break;
    default: o0 = v; o1 = pp; o2 = q; break;
  }
  const float k = float(255.999);                      // convert_image_dtype(float -> uint8): x * (255 + 1 - 1e-3)
  p.c[0] = __float2uint_rz(__fmul_rn(o0, k));
  p.c[1] = __float2uint_rz(__fmul_rn(o1, k));
  p.c[2] = __float2uint_rz(__fmul_rn(o2, k));
}

__device__ __forceinline__ float contrast_mean(const uint64_t* sums, int img, const yb_aug_op& op) {
  const int64_t n = int64_t(op.arg[1]) * op.arg[2];
  return __fdiv_rn(__ull2float_rn(sums[img * YB_AUG_MAX_CONTRAST + op.arg[0]]), __ll2float_rn(n));
}

// The pixel at (y, x) of the image after ops [0, end) of image `img`.
__device__ Rgb pixel_at(const yb_aug_image& d, int img, int end, int y, int x, const uint64_t* sums) {
  Rgb p;
  int origin = 0;
  for (int k = end - 1; k >= 0; --k) {
    const int kind = d.ops[k].kind;
    if (kind == YB_AUG_HFLIP) {
      x = d.ops[k].arg[0] - 1 - x;
    } else if (kind == YB_AUG_CROP) {
      y += d.ops[k].arg[0];
      x += d.ops[k].arg[1];
    } else if (kind == YB_AUG_ZOOM_OUT) {
      y -= d.ops[k].arg[0];
      x -= d.ops[k].arg[1];
      if (y < 0 || x < 0 || y >= d.ops[k].arg[2] || x >= d.ops[k].arg[3]) {
        const uint32_t fill = uint32_t(d.ops[k].arg[6]);
        p.c[0] = fill & 255u;
        p.c[1] = (fill >> 8) & 255u;
        p.c[2] = (fill >> 16) & 255u;
        origin = k + 1;
        break;
      }
    }
  }
  if (origin == 0) {
    const uint8_t* s = d.src + int64_t(y) * d.stride_y + int64_t(x) * d.stride_x;
    p.c[0] = __ldg(s);
    p.c[1] = __ldg(s + d.stride_c);
    p.c[2] = __ldg(s + 2 * d.stride_c);
  }
  for (int k = origin; k < end; ++k) {
    const yb_aug_op& op = d.ops[k];
    switch (op.kind) {
      case YB_AUG_BRIGHTNESS:
#pragma unroll
        for (int c = 0; c < 3; ++c) p.c[c] = blend(p.c[c], 0.0f, op.factor, op.one_minus);
        break;
      case YB_AUG_CONTRAST: {
        const float m = contrast_mean(sums, img, op);
#pragma unroll
        for (int c = 0; c < 3; ++c) p.c[c] = blend(p.c[c], m, op.factor, op.one_minus);
        break;
      }
      case YB_AUG_SATURATION: {
        const float gr = __uint2float_rn(gray(p));
#pragma unroll
        for (int c = 0; c < 3; ++c) p.c[c] = blend(p.c[c], gr, op.factor, op.one_minus);
        break;
      }
      case YB_AUG_HUE:
        hue(p, op.factor);
        break;
      case YB_AUG_PERMUTE: {
        const Rgb q = p;
#pragma unroll
        for (int c = 0; c < 3; ++c) p.c[c] = op.arg[c] == 0 ? q.c[0] : op.arg[c] == 1 ? q.c[1] : q.c[2];
        break;
      }
      default:
        break;
    }
  }
  return p;
}

// The image whose [start, start + blocks) holds block b: the last image with start <= b (images without blocks share
// their successor's start).
template <typename Start>
__device__ __forceinline__ int find_image(const yb_aug_image* imgs, int n, int b, Start start) {
  int lo = 0, hi = n;                                   // first image with start > b
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (start(imgs[mid]) <= b) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

__global__ void __launch_bounds__(kThreads) augment_mean_kernel(const yb_aug_image* __restrict__ imgs, int n,
                                                                int round, uint64_t* __restrict__ sums) {
  const int b = int(blockIdx.x);
  const int i = find_image(imgs, n, b, [round](const yb_aug_image& d) { return d.mean_block_start[round]; });
  const yb_aug_image& d = imgs[i];
  int k = 0;                                            // the op of this round
  for (int r = -1; k < d.n_ops; ++k)
    if (d.ops[k].kind == YB_AUG_CONTRAST && ++r == round) break;
  const int w = d.ops[k].arg[2];
  const int64_t total = int64_t(d.ops[k].arg[1]) * w;
  const int64_t base = int64_t(b - d.mean_block_start[round]) * kBlockPix;
  uint32_t acc = 0;
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    const int64_t p = base + int64_t(j) * kThreads + threadIdx.x;
    if (p < total) acc += gray(pixel_at(d, i, k, int(p / w), int(p % w), sums));
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ uint32_t warp_sum[kThreads / 32];
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t s = 0;
    for (int j = 0; j < kThreads / 32; ++j) s += warp_sum[j];
    atomicAdd(reinterpret_cast<unsigned long long*>(&sums[i * YB_AUG_MAX_CONTRAST + round]),
              static_cast<unsigned long long>(s));
  }
}

template <typename T>
__device__ __forceinline__ T out_value(uint32_t byte);
template <>
__device__ __forceinline__ uint8_t out_value<uint8_t>(uint32_t byte) { return uint8_t(byte); }
template <>
__device__ __forceinline__ float out_value<float>(uint32_t byte) { return __fdiv_rn(__uint2float_rn(byte), 255.0f); }

template <typename T>
__device__ __forceinline__ void store4(T* dst, const T (&v)[kPix]);
template <>
__device__ __forceinline__ void store4<uint8_t>(uint8_t* dst, const uint8_t (&v)[kPix]) {
  *reinterpret_cast<uchar4*>(dst) = make_uchar4(v[0], v[1], v[2], v[3]);
}
template <>
__device__ __forceinline__ void store4<float>(float* dst, const float (&v)[kPix]) {
  *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) augment_output_kernel(const yb_aug_image* __restrict__ imgs, int n,
                                                                  const uint64_t* __restrict__ sums, T* __restrict__ out) {
  const int b = int(blockIdx.x);
  const int i = find_image(imgs, n, b, [](const yb_aug_image& d) { return d.out_block_start; });
  const yb_aug_image& d = imgs[i];
  const int w = d.out_w;
  const int64_t plane = int64_t(d.out_h) * w;
  const int64_t p0 = int64_t(b - d.out_block_start) * kBlockPix + int64_t(threadIdx.x) * kPix;
  if (p0 >= plane) return;
  int y = int(p0 / w), x = int(p0 % w);
  T v[3][kPix];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (p0 + j < plane) {
      const Rgb p = pixel_at(d, i, d.n_ops, y, x, sums);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c][j] = out_value<T>(p.c[c]);
    }
    if (++x == w) {
      x = 0;
      ++y;
    }
  }
  T* base = out + d.out_offset + p0;
  const bool full = p0 + kPix <= plane;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    T* dst = base + c * plane;
    if (full && (reinterpret_cast<uintptr_t>(dst) % (kPix * sizeof(T))) == 0) {
      store4<T>(dst, v[c]);
    } else {
#pragma unroll
      for (int j = 0; j < kPix; ++j)
        if (p0 + j < plane) dst[j] = v[c][j];
    }
  }
}

int64_t blocks_for(int64_t pixels) { return (pixels + kBlockPix - 1) / kBlockPix; }

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_augment_prepare(int n_images, yb_aug_image* images, int64_t* totals) {
  YB_REQUIRE(n_images > 0 && images && totals, "augment_prepare: null argument or empty batch");
  int64_t out_blocks = 0, mean_blocks[YB_AUG_MAX_CONTRAST] = {0, 0, 0, 0};
  for (int i = 0; i < n_images; ++i) {
    yb_aug_image& d = images[i];
    YB_REQUIRE(d.src && d.src_h > 0 && d.src_w > 0, "augment_prepare: image %d has no pixels", i);
    YB_REQUIRE(d.n_ops >= 0 && d.n_ops <= YB_AUG_MAX_OPS, "augment_prepare: image %d has %d ops (at most %d)", i,
               d.n_ops, YB_AUG_MAX_OPS);
    int64_t h = d.src_h, w = d.src_w;
    int rounds = 0;
    for (int r = 0; r < YB_AUG_MAX_CONTRAST; ++r) d.mean_block_start[r] = int32_t(mean_blocks[r]);
    for (int k = 0; k < d.n_ops; ++k) {
      yb_aug_op& op = d.ops[k];
      switch (op.kind) {
        case YB_AUG_BRIGHTNESS:
        case YB_AUG_SATURATION:
        case YB_AUG_HUE:
          break;
        case YB_AUG_CONTRAST:
          YB_REQUIRE(rounds < YB_AUG_MAX_CONTRAST, "augment_prepare: image %d has more than %d contrast ops", i,
                     YB_AUG_MAX_CONTRAST);
          YB_REQUIRE(op.arg[1] == h && op.arg[2] == w, "augment_prepare: image %d op %d: contrast size mismatch", i, k);
          op.arg[0] = rounds;
          mean_blocks[rounds] += blocks_for(h * w);
          ++rounds;
          break;
        case YB_AUG_PERMUTE:
          for (int c = 0; c < 3; ++c)
            YB_REQUIRE(op.arg[c] >= 0 && op.arg[c] < 3, "augment_prepare: image %d op %d: bad permutation", i, k);
          break;
        case YB_AUG_ZOOM_OUT:
          YB_REQUIRE(op.arg[2] == h && op.arg[3] == w && op.arg[0] >= 0 && op.arg[1] >= 0 &&
                         op.arg[0] + h <= op.arg[4] && op.arg[1] + w <= op.arg[5],
                     "augment_prepare: image %d op %d: zoom-out does not hold the image", i, k);
          h = op.arg[4];
          w = op.arg[5];
          break;
        case YB_AUG_CROP:
          YB_REQUIRE(op.arg[0] >= 0 && op.arg[1] >= 0 && op.arg[2] > 0 && op.arg[3] > 0 && op.arg[0] + op.arg[2] <= h &&
                         op.arg[1] + op.arg[3] <= w,
                     "augment_prepare: image %d op %d: crop outside the image", i, k);
          h = op.arg[2];
          w = op.arg[3];
          break;
        case YB_AUG_HFLIP:
          YB_REQUIRE(op.arg[0] == w, "augment_prepare: image %d op %d: flip width mismatch", i, k);
          break;
        default:
          YB_REQUIRE(false, "augment_prepare: image %d op %d has unknown kind %d", i, k, op.kind);
      }
      YB_REQUIRE(h < (1 << 20) && w < (1 << 20), "augment_prepare: image %d grows beyond 2^20 pixels a side", i);
    }
    d.n_contrast = rounds;
    YB_REQUIRE(d.out_h == h && d.out_w == w, "augment_prepare: image %d: output %dx%d, the ops give %lldx%lld", i,
               d.out_h, d.out_w, (long long)h, (long long)w);
    d.out_block_start = int32_t(out_blocks);
    out_blocks += blocks_for(h * w);
    YB_REQUIRE(out_blocks < (int64_t(1) << 31), "augment_prepare: batch too large");
  }
  totals[0] = out_blocks;
  for (int r = 0; r < YB_AUG_MAX_CONTRAST; ++r) totals[1 + r] = mean_blocks[r];
  return YB_OK;
}

extern "C" int yb_augment(int n_images, const yb_aug_image* images_host, const yb_aug_image* images_dev,
                          void* out_dev, int32_t out_dtype, uint64_t* sums_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(n_images > 0 && images_host && images_dev && out_dev && sums_dev, "augment: null argument");
  YB_REQUIRE(out_dtype == YB_U8 || out_dtype == YB_F32, "augment: output dtype %d (uint8 or float32)", out_dtype);
  int64_t out_blocks = 0, mean_blocks[YB_AUG_MAX_CONTRAST] = {0, 0, 0, 0};
  int rounds = 0;
  for (int i = 0; i < n_images; ++i) {
    const yb_aug_image& d = images_host[i];
    out_blocks += blocks_for(int64_t(d.out_h) * d.out_w);
    rounds = rounds > d.n_contrast ? rounds : d.n_contrast;
    for (int k = 0; k < d.n_ops; ++k)
      if (d.ops[k].kind == YB_AUG_CONTRAST) mean_blocks[d.ops[k].arg[0]] += blocks_for(int64_t(d.ops[k].arg[1]) * d.ops[k].arg[2]);
  }
  if (rounds > 0) {
    YB_CHECK_CUDA(cudaMemsetAsync(sums_dev, 0, sizeof(uint64_t) * size_t(n_images) * YB_AUG_MAX_CONTRAST, stream));
    for (int r = 0; r < rounds; ++r) {
      augment_mean_kernel<<<unsigned(mean_blocks[r]), kThreads, 0, stream>>>(images_dev, n_images, r, sums_dev);
      YB_CHECK_CUDA(cudaGetLastError());
    }
  }
  if (out_blocks == 0) return YB_OK;
  if (out_dtype == YB_U8)
    augment_output_kernel<uint8_t><<<unsigned(out_blocks), kThreads, 0, stream>>>(images_dev, n_images, sums_dev,
                                                                                 static_cast<uint8_t*>(out_dev));
  else
    augment_output_kernel<float><<<unsigned(out_blocks), kThreads, 0, stream>>>(images_dev, n_images, sums_dev,
                                                                               static_cast<float*>(out_dev));
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
