// The two memory-bound ops of MobileNetV3 (yolort/models/yolo_lite.py, torchvision mobilenetv3.py InvertedResidual):
//
//  * YB_OP_DWCONV: depthwise k x k convolution (k = 1, 3, 5; stride 1 or 2; zero padding k / 2), bias + ReLU /
//    Hardswish / linear in fp32, one rounding.  A thread owns one 16-byte channel octet of kPix horizontally adjacent
//    output pixels: per filter row it loads the input octets of the span those pixels read once (neighbouring pixels
//    share k - stride of them), and the k x k weight octets of its channels stay in registers.  Consecutive threads
//    take consecutive octets of the same pixels, so every load and store is a whole 16-byte vector of a contiguous run.
//  * YB_OP_SE: in-place squeeze-excitation, x <- x * hardsigmoid(W2 relu(W1 mean_hw(x) + b1) + b2) per image.  One
//    launch; a thread-block cluster of kSeCtas CTAs per image:
//      1. each CTA sums its own range of pixels per channel in fp32 (fixed order: a thread owns one channel octet and
//         one pixel lane, the lanes are added in lane order),
//      2. the CTAs exchange those partial sums through distributed shared memory and every CTA adds them in rank
//         order, so all of them hold the same mean, bit for bit,
//      3. every CTA computes the gate itself (at most C x S + S x C MACs, fp32 weights from L2),
//      4. each CTA scales its own pixel range, which it read moments earlier (mostly L2 hits).
//    No atomics, no workspace: a repeated run and a graph replay give the same bits.
// Both kernels use programmatic dependent launch like the convolutions: they wait for the previous launch before
// touching activations.
#include <cooperative_groups.h>

#include "common.cuh"
#include "conv_epilogue.cuh"
#include "conv_sm90.h"

namespace cg = cooperative_groups;

namespace yb {

namespace {

constexpr int kDwThreads = 256;
constexpr int kDwPix = 4;                   // output pixels per thread along x
constexpr int kSeThreads = 256;
constexpr int kSeCtas = 8;                  // cluster size: CTAs per image (portable maximum)
constexpr int kSeMaxC = 2048;
constexpr int kSeMaxS = 1024;

struct DwParams {
  const uint16_t* in;
  uint16_t* out;
  const uint16_t* w;    // [k*k][C]
  const float* b;       // [C]
  int N, H, W, Ho, Wo, C, in_cs, out_cs, act;
  int xgroups;          // ceil(Wo / kDwPix)
};

template <bool kBf16>
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = unpack2<kBf16>(u[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__device__ __forceinline__ float act_fn(float v, int act) {
  if (act == YB_ACT_RELU) return fmaxf(v, 0.f);
  if (act == YB_ACT_HARDSWISH) return v * fminf(fmaxf(v + 3.0f, 0.f), 6.0f) * (1.0f / 6.0f);
  return v;
}

// grid: ceil(N * Ho * xgroups * C/8 / 256); thread -> (image, output row, group of kDwPix columns, channel octet)
template <bool kBf16, int kK, int kS>
__global__ void __launch_bounds__(kDwThreads) dwconv_kernel(const DwParams p) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c8n = p.C >> 3;
  const long long total = static_cast<long long>(p.N) * p.Ho * p.xgroups * c8n;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8 = static_cast<int>(idx % c8n);
  long long t = idx / c8n;
  const int xg = static_cast<int>(t % p.xgroups);
  t /= p.xgroups;
  const int y = static_cast<int>(t % p.Ho);
  const int n = static_cast<int>(t / p.Ho);
  constexpr int s = kS;
  constexpr int pad = kK / 2;
  const int x0 = xg * kDwPix;

  float acc[kDwPix][8];
  {
    float bias[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bias[j] = __ldg(p.b + c8 * 8 + j);
#pragma unroll
    for (int q = 0; q < kDwPix; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[q][j] = bias[j];
  }
  const uint16_t* img = p.in + static_cast<long long>(n) * p.H * p.W * p.in_cs + c8 * 8;
  // input columns read by the kDwPix outputs: x0*s - pad .. (x0 + kDwPix - 1)*s - pad + kK - 1
  constexpr int kSpan = (kDwPix - 1) * kS + kK;
  const int xi0 = x0 * s - pad;
#pragma unroll
  for (int i = 0; i < kK; ++i) {
    const int yy = y * s - pad + i;
    if (yy < 0 || yy >= p.H) continue;
    float wv[kK][8];
#pragma unroll
    for (int j = 0; j < kK; ++j)
      unpack8<kBf16>(__ldg(reinterpret_cast<const uint4*>(p.w + (i * kK + j) * p.C + c8 * 8)), wv[j]);
    const uint16_t* row = img + static_cast<long long>(yy) * p.W * p.in_cs;
#pragma unroll
    for (int r = 0; r < kSpan; ++r) {
      const int xx = xi0 + r;
      if (xx < 0 || xx >= p.W) continue;
      float v[8];
      unpack8<kBf16>(__ldg(reinterpret_cast<const uint4*>(row + static_cast<long long>(xx) * p.in_cs)), v);
#pragma unroll
      for (int q = 0; q < kDwPix; ++q) {
        const int j = r - q * s;          // tap of output pixel x0 + q that reads input column xi0 + r
        if (j >= 0 && j < kK) {
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[q][e] = fmaf(wv[j][e], v[e], acc[q][e]);
        }
      }
    }
  }
  uint16_t* orow = p.out + (static_cast<long long>(n) * p.Ho + y) * p.Wo * p.out_cs + c8 * 8;
#pragma unroll
  for (int q = 0; q < kDwPix; ++q) {
    const int x = x0 + q;
    if (x >= p.Wo) break;
    uint4 o;
    uint32_t* u = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) u[e] = pack2<kBf16>(act_fn(acc[q][2 * e], p.act), act_fn(acc[q][2 * e + 1], p.act));
    *reinterpret_cast<uint4*>(orow + static_cast<long long>(x) * p.out_cs) = o;
  }
}

struct SeParams {
  uint16_t* x;
  const float* w1t;   // [C][S]
  const float* w2t;   // [S][C]
  const float* b1;    // [S]
  const float* b2;    // [C]
  int HW, C, S, cs;
};

// grid: (kSeCtas, N), cluster (kSeCtas, 1, 1); CTA rank r of image n owns pixels [r*per, min(HW, (r+1)*per)).
template <bool kBf16>
__global__ void __launch_bounds__(kSeThreads) se_kernel(const SeParams p) {
  __shared__ float part[kSeMaxC];     // per-lane partial sums (lanes x C <= kSeMaxC), then this CTA's sums
  __shared__ float csum[kSeMaxC];     // this CTA's channel sums; after the exchange, the gate
  __shared__ float mean[kSeMaxC];
  __shared__ float hidden[kSeMaxS];
  cg::cluster_group cluster = cg::this_cluster();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int rank = static_cast<int>(cluster.block_rank());
  const int n = blockIdx.y;
  const int C = p.C, C8 = C >> 3;
  const int per = (p.HW + kSeCtas - 1) / kSeCtas;
  const int p0 = min(p.HW, rank * per), p1 = min(p.HW, p0 + per);
  uint16_t* img = p.x + static_cast<long long>(n) * p.HW * p.cs;
  const int lanes = C8 >= kSeThreads ? 1 : kSeThreads / C8;

  // 1. partial sums: item = (lane, octet); lane l adds pixels p0 + l, p0 + l + lanes, ... in order
  for (int item = threadIdx.x; item < lanes * C8; item += kSeThreads) {
    const int c8 = item % C8, lane = item / C8;
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int px = p0 + lane; px < p1; px += lanes) {
      float v[8];
      unpack8<kBf16>(*reinterpret_cast<const uint4*>(img + static_cast<long long>(px) * p.cs + c8 * 8), v);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += v[e];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) part[lane * C + c8 * 8 + e] = a[e];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kSeThreads) {
    float a = 0.f;
    for (int l = 0; l < lanes; ++l) a += part[l * C + c];
    csum[c] = a;
  }
  // 2. exchange through distributed shared memory, summed in rank order
  cluster.sync();
  const float inv = 1.0f / static_cast<float>(p.HW);
  for (int c = threadIdx.x; c < C; c += kSeThreads) {
    float a = 0.f;
#pragma unroll
    for (int r = 0; r < kSeCtas; ++r) a += cluster.map_shared_rank(csum, r)[c];
    mean[c] = a * inv;
  }
  cluster.sync();   // every CTA has read every csum: csum may be reused and no CTA exits while it is read
  // 3. gate
  for (int j = threadIdx.x; j < p.S; j += kSeThreads) {
    float h = __ldg(p.b1 + j);
    for (int c = 0; c < C; ++c) h = fmaf(__ldg(p.w1t + static_cast<long long>(c) * p.S + j), mean[c], h);
    hidden[j] = fmaxf(h, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kSeThreads) {
    float g = __ldg(p.b2 + c);
    for (int j = 0; j < p.S; ++j) g = fmaf(__ldg(p.w2t + static_cast<long long>(j) * C + c), hidden[j], g);
    csum[c] = fminf(fmaxf(g + 3.0f, 0.f), 6.0f) / 6.0f;
  }
  __syncthreads();
  // 4. scale this CTA's pixels
  const long long items = static_cast<long long>(p1 - p0) * C8;
  for (long long it = threadIdx.x; it < items; it += kSeThreads) {
    const int px = p0 + static_cast<int>(it / C8), c8 = static_cast<int>(it % C8);
    uint4* ptr = reinterpret_cast<uint4*>(img + static_cast<long long>(px) * p.cs + c8 * 8);
    float v[8];
    unpack8<kBf16>(*ptr, v);
    uint4 o;
    uint32_t* u = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) u[e] = pack2<kBf16>(v[2 * e] * csum[c8 * 8 + 2 * e], v[2 * e + 1] * csum[c8 * 8 + 2 * e + 1]);
    *ptr = o;
  }
}

bool aligned(const void* ptr, uintptr_t a) { return (reinterpret_cast<uintptr_t>(ptr) & (a - 1)) == 0; }

}  // namespace

int dwconv_configure_check(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "dwconv: dtype must be f16 or bf16");
  YB_REQUIRE(d.residual == nullptr && d.decode == nullptr && d.chain == nullptr,
             "dwconv: residual, decode and chain must be NULL");
  YB_REQUIRE(d.reserved == 0, "dwconv: reserved must be 0, got 0x%x", d.reserved);
  YB_REQUIRE(d.weight != nullptr && d.bias != nullptr, "dwconv: null weight or bias");
  YB_REQUIRE(d.ksize == 1 || d.ksize == 3 || d.ksize == 5, "dwconv: ksize must be 1, 3 or 5, got %d", d.ksize);
  YB_REQUIRE(d.stride == 1 || d.stride == 2, "dwconv: stride must be 1 or 2, got %d", d.stride);
  YB_REQUIRE(d.pad == d.ksize / 2, "dwconv: pad must be ksize/2 = %d, got %d", d.ksize / 2, d.pad);
  YB_REQUIRE(d.act == YB_ACT_NONE || d.act == YB_ACT_RELU || d.act == YB_ACT_HARDSWISH,
             "dwconv: act must be NONE, RELU or HARDSWISH, got %d", d.act);
  YB_REQUIRE(d.Cin == d.Cout, "dwconv: Cin (%d) must equal Cout (%d)", d.Cin, d.Cout);
  YB_REQUIRE(d.Cin > 0 && d.Cin % 8 == 0 && d.in_cstride % 8 == 0 && d.in_cstride >= d.Cin && d.out_cstride % 8 == 0 &&
                 d.out_cstride >= d.Cout,
             "dwconv: C and the channel strides must be multiples of 8 with cstride >= C, got %d/%d/%d", d.Cin,
             d.in_cstride, d.out_cstride);
  YB_REQUIRE(d.N >= 1 && d.H >= 1 && d.W >= 1, "dwconv: empty input (N=%d H=%d W=%d)", d.N, d.H, d.W);
  const int ho = (d.H + 2 * d.pad - d.ksize) / d.stride + 1, wo = (d.W + 2 * d.pad - d.ksize) / d.stride + 1;
  YB_REQUIRE(d.Ho == ho && d.Wo == wo, "dwconv: output extent (%d,%d) must be (%d,%d)", d.Ho, d.Wo, ho, wo);
  YB_REQUIRE(aligned(d.in, 16) && aligned(d.out, 16) && aligned(d.weight, 16) && aligned(d.bias, 4),
             "dwconv: in, out and weight must be 16-byte aligned, bias 4-byte aligned");
  return YB_OK;
}

int se_configure_check(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "se: dtype must be f16 or bf16");
  YB_REQUIRE(d.residual == nullptr && d.decode == nullptr && d.chain == nullptr,
             "se: residual, decode and chain must be NULL");
  YB_REQUIRE(d.reserved == 0, "se: reserved must be 0, got 0x%x", d.reserved);
  YB_REQUIRE(d.weight != nullptr && d.bias != nullptr, "se: null weight or bias");
  YB_REQUIRE(d.in == d.out && d.in_cstride == d.out_cstride, "se: works in place: in must equal out (and the strides)");
  YB_REQUIRE(d.Cin == d.Cout, "se: Cin (%d) must equal Cout (%d)", d.Cin, d.Cout);
  YB_REQUIRE(d.Cin > 0 && d.Cin % 8 == 0 && d.Cin <= kSeMaxC && d.in_cstride % 8 == 0 && d.in_cstride >= d.Cin,
             "se: C must be a multiple of 8 up to %d and in_cstride a multiple of 8 >= C, got %d/%d", kSeMaxC, d.Cin,
             d.in_cstride);
  YB_REQUIRE(d.ksize >= 1 && d.ksize <= kSeMaxS, "se: ksize holds the squeeze width, 1..%d, got %d", kSeMaxS, d.ksize);
  YB_REQUIRE(d.N >= 1 && d.N <= 65535 && d.H >= 1 && d.W >= 1, "se: empty or too large input (N=%d H=%d W=%d)", d.N,
             d.H, d.W);
  YB_REQUIRE(d.Ho == d.H && d.Wo == d.W, "se: output extent must equal the input extent");
  YB_REQUIRE(static_cast<long long>(d.H) * d.W < (1ll << 31), "se: map too large");
  YB_REQUIRE(aligned(d.in, 16) && aligned(d.weight, 16) && aligned(d.bias, 16),
             "se: tensor, weight and bias must be 16-byte aligned");
  return YB_OK;
}

int dwconv_launch(const yb_op_desc& d, cudaStream_t stream) {
  DwParams p;
  p.in = static_cast<const uint16_t*>(d.in);
  p.out = static_cast<uint16_t*>(d.out);
  p.w = static_cast<const uint16_t*>(d.weight);
  p.b = d.bias;
  p.N = d.N, p.H = d.H, p.W = d.W, p.Ho = d.Ho, p.Wo = d.Wo, p.C = d.Cin;
  p.in_cs = d.in_cstride, p.out_cs = d.out_cstride, p.act = d.act;
  p.xgroups = (d.Wo + kDwPix - 1) / kDwPix;
  const long long total = static_cast<long long>(d.N) * d.Ho * p.xgroups * (d.Cin >> 3);
  using Fn = void (*)(const DwParams);
  static const Fn table[2][3][2] = {
      {{dwconv_kernel<false, 1, 1>, dwconv_kernel<false, 1, 2>}, {dwconv_kernel<false, 3, 1>, dwconv_kernel<false, 3, 2>},
       {dwconv_kernel<false, 5, 1>, dwconv_kernel<false, 5, 2>}},
      {{dwconv_kernel<true, 1, 1>, dwconv_kernel<true, 1, 2>}, {dwconv_kernel<true, 3, 1>, dwconv_kernel<true, 3, 2>},
       {dwconv_kernel<true, 5, 1>, dwconv_kernel<true, 5, 2>}}};
  const Fn fn = table[d.dtype == YB_BF16 ? 1 : 0][d.ksize / 2][d.stride - 1];
  YB_CHECK_CUDA(launch_pdl(fn, dim3(static_cast<unsigned>((total + kDwThreads - 1) / kDwThreads)), dim3(kDwThreads), 0, stream, p));
  return YB_OK;
}

int se_launch(const yb_op_desc& d, cudaStream_t stream) {
  SeParams p;
  p.x = static_cast<uint16_t*>(d.out);
  p.C = d.Cin, p.S = d.ksize, p.cs = d.in_cstride, p.HW = d.H * d.W;
  p.w1t = static_cast<const float*>(d.weight);
  p.w2t = p.w1t + static_cast<long long>(p.C) * p.S;
  p.b1 = d.bias;
  p.b2 = d.bias + p.S;
  YB_CHECK_CUDA(launch_pdl_cluster(kSeCtas, d.dtype == YB_BF16 ? se_kernel<true> : se_kernel<false>,
                                   dim3(kSeCtas, static_cast<unsigned>(d.N)), dim3(kSeThreads), 0, stream, p));
  return YB_OK;
}

}  // namespace yb
