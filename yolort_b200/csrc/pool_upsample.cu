// HBM-bound neck helpers on NHWC fp16/bf16 slices.
//
//  * SPP pooling (yolort/v5/models/common.py:176-187, instantiated at
//    yolort/models/path_aggregation_network.py:109-110 with k=(5,9,13)): max-pools of window 5/9/13,
//    stride 1, implicit -inf padding, written next to the input inside the concat buffer:
//    channels [C,2C) = mp5, [2C,3C) = mp9, [3C,4C) = mp13.  One pass over a 13x13 neighbourhood
//    produces all three (nested windows), 8 channels (16 bytes) per thread.
//  * nearest-neighbour 2x upsample (nn.Upsample(scale_factor=2), path_aggregation_network.py:123,134),
//    writing into a channel window of the next concat buffer.
#include "common.cuh"
#include "conv_sm90.h"

namespace yb {
namespace {

template <bool kBf16>
__device__ __forceinline__ void max8(uint4& acc, const uint4& v) {
  if constexpr (kBf16) {
    __nv_bfloat162* a = reinterpret_cast<__nv_bfloat162*>(&acc);
    const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = __hmax2(a[i], b[i]);
  } else {
    __half2* a = reinterpret_cast<__half2*>(&acc);
    const __half2* b = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = __hmax2(a[i], b[i]);
  }
}

// grid: (ceil(N*H*W*C8 / 256)); thread -> (pixel, channel octet)
template <bool kBf16>
__global__ void spp_pool_kernel(const uint16_t* __restrict__ in, int in_cs, uint16_t* __restrict__ out,
                                int out_cs, int N, int H, int W, int C) {
  const int c8n = C >> 3;
  const long long total = static_cast<long long>(N) * H * W * c8n;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8 = static_cast<int>(idx % c8n);
  long long pix = idx / c8n;
  const int x = static_cast<int>(pix % W);
  pix /= W;
  const int y = static_cast<int>(pix % H);
  const int n = static_cast<int>(pix / H);
  const uint32_t ninf2 = kBf16 ? 0xFF80FF80u : 0xFC00FC00u;  // (-inf, -inf)
  uint4 m5 = make_uint4(ninf2, ninf2, ninf2, ninf2), m9 = m5, m13 = m5;
  const uint16_t* base = in + static_cast<long long>(n) * H * W * in_cs + c8 * 8;
  for (int dy = -6; dy <= 6; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    const int ady = dy < 0 ? -dy : dy;
    for (int dx = -6; dx <= 6; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      const int adx = dx < 0 ? -dx : dx;
      const int r = ady > adx ? ady : adx;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + (static_cast<long long>(yy) * W + xx) * in_cs));
      max8<kBf16>(m13, v);
      if (r <= 4) max8<kBf16>(m9, v);
      if (r <= 2) max8<kBf16>(m5, v);
    }
  }
  uint16_t* o = out + ((static_cast<long long>(n) * H + y) * W + x) * out_cs + c8 * 8;
  *reinterpret_cast<uint4*>(o) = m5;
  *reinterpret_cast<uint4*>(o + C) = m9;
  *reinterpret_cast<uint4*>(o + 2 * C) = m13;
}

// SPPF-style cascade in shared memory: mp9 = mp5(mp5(x)), mp13 = mp5(mp9) (exactly equal to the direct
// windows with -inf padding, yolort/v5/models/common.py:196).  One CTA owns the H x W planes of G adjacent channel
// octets of one image: 3 buffers of H*W*G 16-byte items [pixel][octet] in shared memory, separable 5-tap max (rows then
// columns).  G octets = 16 G contiguous bytes per pixel in global memory (whole 32-byte sectors from G = 2).
template <bool kBf16>
__global__ void spp_pool_cascade_kernel(const uint16_t* __restrict__ in, int in_cs, uint16_t* __restrict__ out,
                                        int out_cs, int H, int W, int C, int G) {
  extern __shared__ __align__(16) uint8_t pool_smem[];
  const int groups = (C >> 3) / G;
  const int n = blockIdx.x / groups;
  const int c8 = (blockIdx.x - n * groups) * G;      // first octet of this CTA
  const int HW = H * W, items = HW * G;
  uint4* cur = reinterpret_cast<uint4*>(pool_smem);
  uint4* tmp = cur + items;
  uint4* nxt = tmp + items;
  const uint16_t* src = in + static_cast<long long>(n) * HW * in_cs + c8 * 8;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int pix = i / G, o = i - pix * G;
    cur[i] = __ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(pix) * in_cs + o * 8));
  }
  __syncthreads();
  uint16_t* dst = out + static_cast<long long>(n) * HW * out_cs + c8 * 8;
  for (int level = 0; level < 3; ++level) {
    for (int i = threadIdx.x; i < items; i += blockDim.x) {  // horizontal 5-tap
      const int pix = i / G;
      const int y = pix / W, x = pix - y * W;
      uint4 m = cur[i];
      for (int dx = -2; dx <= 2; ++dx) {
        const int xx = x + dx;
        if (dx != 0 && xx >= 0 && xx < W) max8<kBf16>(m, cur[i + dx * G]);
      }
      tmp[i] = m;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < items; i += blockDim.x) {  // vertical 5-tap
      const int pix = i / G, o = i - pix * G;
      const int y = pix / W;
      uint4 m = tmp[i];
      for (int dy = -2; dy <= 2; ++dy) {
        const int yy = y + dy;
        if (dy != 0 && yy >= 0 && yy < H) max8<kBf16>(m, tmp[i + dy * W * G]);
      }
      nxt[i] = m;
      *reinterpret_cast<uint4*>(dst + static_cast<long long>(pix) * out_cs + level * C + o * 8) = m;
    }
    __syncthreads();
    uint4* t = cur;
    cur = nxt;
    nxt = t;
  }
}

__global__ void upsample2x_kernel(const uint16_t* __restrict__ in, int in_cs, uint16_t* __restrict__ out,
                                  int out_cs, int N, int H, int W, int C) {
  const int c8n = C >> 3;
  const int Ho = 2 * H, Wo = 2 * W;
  const long long total = static_cast<long long>(N) * Ho * Wo * c8n;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8 = static_cast<int>(idx % c8n);
  long long pix = idx / c8n;
  const int x = static_cast<int>(pix % Wo);
  pix /= Wo;
  const int y = static_cast<int>(pix % Ho);
  const int n = static_cast<int>(pix / Ho);
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(
      in + ((static_cast<long long>(n) * H + (y >> 1)) * W + (x >> 1)) * in_cs + c8 * 8));
  *reinterpret_cast<uint4*>(out + ((static_cast<long long>(n) * Ho + y) * Wo + x) * out_cs + c8 * 8) = v;
}

}  // namespace

int validate_pool_or_upsample(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "pool/upsample: dtype must be f16 or bf16");
  YB_REQUIRE(d.Cin % 8 == 0 && d.in_cstride % 8 == 0 && d.out_cstride % 8 == 0,
             "pool/upsample: channels and strides must be multiples of 8");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(d.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0,
             "pool/upsample: tensors must be 16-byte aligned");
  if (d.kind == YB_OP_SPP_POOL) {
    YB_REQUIRE(d.Ho == d.H && d.Wo == d.W && d.Cout == 3 * d.Cin, "spp_pool: expects Cout == 3*Cin, same extent");
  } else {
    YB_REQUIRE(d.Ho == 2 * d.H && d.Wo == 2 * d.W && d.Cout == d.Cin, "upsample2x: expects doubled extent");
  }
  return YB_OK;
}

int spp_pool_launch(const yb_op_desc& d, cudaStream_t stream) {
  // channel octets per CTA: as many (8, 4, 2, 1) as divide the octet count and fit 3 buffers in shared memory
  // (the kernel is bound by its seven barrier-separated passes per CTA, not by the lines a load touches; two octets keep
  // loads at whole sectors)
  int G = 2;
  while (G > 1 && (((d.Cin >> 3) % G) != 0 || static_cast<size_t>(d.H) * d.W * 16 * 3 * G > 200 * 1024)) G >>= 1;
  const size_t plane_smem = static_cast<size_t>(d.H) * d.W * 16 * 3 * G;
  if (plane_smem <= 200 * 1024) {
    static size_t configured[2] = {48 * 1024, 48 * 1024};
    const int bf = d.dtype == YB_BF16 ? 1 : 0;
    if (plane_smem > configured[bf]) {
      if (bf)
        YB_CHECK_CUDA(cudaFuncSetAttribute(spp_pool_cascade_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(plane_smem)));
      else
        YB_CHECK_CUDA(cudaFuncSetAttribute(spp_pool_cascade_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(plane_smem)));
      configured[bf] = plane_smem;
    }
    const unsigned blocks = static_cast<unsigned>(d.N) * ((d.Cin >> 3) / G);
    const int threads = G >= 4 ? 512 : 256;
    if (bf)
      spp_pool_cascade_kernel<true><<<blocks, threads, plane_smem, stream>>>(
          static_cast<const uint16_t*>(d.in), d.in_cstride, static_cast<uint16_t*>(d.out), d.out_cstride, d.H, d.W, d.Cin, G);
    else
      spp_pool_cascade_kernel<false><<<blocks, threads, plane_smem, stream>>>(
          static_cast<const uint16_t*>(d.in), d.in_cstride, static_cast<uint16_t*>(d.out), d.out_cstride, d.H, d.W, d.Cin, G);
    YB_CHECK_CUDA(cudaGetLastError());
    return YB_OK;
  }
  // very large planes: direct 13x13 window per thread
  const long long total = static_cast<long long>(d.N) * d.H * d.W * (d.Cin >> 3);
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
  if (d.dtype == YB_BF16)
    spp_pool_kernel<true><<<blocks, threads, 0, stream>>>(
        static_cast<const uint16_t*>(d.in), d.in_cstride, static_cast<uint16_t*>(d.out), d.out_cstride,
        d.N, d.H, d.W, d.Cin);
  else
    spp_pool_kernel<false><<<blocks, threads, 0, stream>>>(
        static_cast<const uint16_t*>(d.in), d.in_cstride, static_cast<uint16_t*>(d.out), d.out_cstride,
        d.N, d.H, d.W, d.Cin);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

int upsample2x_launch(const yb_op_desc& d, cudaStream_t stream) {
  const long long total = static_cast<long long>(d.N) * d.Ho * d.Wo * (d.Cin >> 3);
  const int threads = 256;
  const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
  upsample2x_kernel<<<blocks, threads, 0, stream>>>(static_cast<const uint16_t*>(d.in), d.in_cstride,
                                                    static_cast<uint16_t*>(d.out), d.out_cstride, d.N,
                                                    d.H, d.W, d.Cin);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

}  // namespace yb
