// YB_OP_AVGPOOL: global average pool (nn.AdaptiveAvgPool2d(1) of the DarkNet classifiers, yolort/models/darknetv4.py,
// darknetv6.py) over an NHWC view, out[n, 0, 0, c] = round(sum_px in[n, px, c] / (H * W)).
//
// A CTA owns one image and up to kOcts adjacent 16-byte channel octets.  Thread t takes octet t % octs and pixel lane
// t / octs, so consecutive threads load consecutive octets of the same pixel (one contiguous run of 16 * octs bytes).
// Each lane adds its pixels lane, lane + lanes, ... in order in fp32; the lanes' partial sums go through shared memory
// and one thread per octet adds them in lane order, divides by H * W and rounds once.  The order of every addition is
// fixed by the shape alone: no atomics, and a repeated run gives the same bits.
// Programmatic dependent launch like the other ops: the kernel waits for the previous launch before reading.
#include "common.cuh"
#include "conv_epilogue.cuh"
#include "conv_sm90.h"

namespace yb {

namespace {

constexpr int kPoolThreads = 256;
constexpr int kOcts = 32;    // channel octets per CTA (512 contiguous bytes of a pixel)

struct PoolParams {
  const uint16_t* in;
  uint16_t* out;
  int HW, C8, in_cs, out_cs, octs, lanes;
};

// grid: (ceil(C8 / octs), N)
template <bool kBf16>
__global__ void __launch_bounds__(kPoolThreads) avgpool_kernel(const PoolParams p) {
  __shared__ float part[kPoolThreads * 8];       // [lane][octet][8]
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int n = blockIdx.y;
  const int o = threadIdx.x % p.octs, lane = threadIdx.x / p.octs;
  const int c8 = blockIdx.x * p.octs + o;
  const bool active = lane < p.lanes && c8 < p.C8;
  if (active) {
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const uint16_t* src = p.in + static_cast<long long>(n) * p.HW * p.in_cs + c8 * 8;
    for (int px = lane; px < p.HW; px += p.lanes) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(px) * p.in_cs));
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2<kBf16>(u[e]);
        a[2 * e] += f.x;
        a[2 * e + 1] += f.y;
      }
    }
    float* dst = part + (lane * p.octs + o) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) dst[e] = a[e];
  }
  __syncthreads();
  if (threadIdx.x < p.octs && c8 < p.C8) {
    float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int l = 0; l < p.lanes; ++l) {
      const float* src = part + (l * p.octs + o) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) s[e] += src[e];
    }
    const float hw = static_cast<float>(p.HW);
    uint4 r;
    uint32_t* u = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int e = 0; e < 4; ++e) u[e] = pack2<kBf16>(s[2 * e] / hw, s[2 * e + 1] / hw);
    *reinterpret_cast<uint4*>(p.out + static_cast<long long>(n) * p.out_cs + c8 * 8) = r;
  }
}

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

}  // namespace

int avgpool_configure_check(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "avgpool: dtype must be f16 or bf16");
  YB_REQUIRE(d.weight == nullptr && d.bias == nullptr && d.residual == nullptr && d.decode == nullptr &&
                 d.chain == nullptr,
             "avgpool: weight, bias, residual, decode and chain must be NULL");
  YB_REQUIRE(d.act == YB_ACT_NONE, "avgpool: act must be 0, got %d", d.act);
  YB_REQUIRE(d.reserved == 0, "avgpool: reserved must be 0, got 0x%x", d.reserved);
  YB_REQUIRE(d.Cin == d.Cout, "avgpool: Cin (%d) must equal Cout (%d)", d.Cin, d.Cout);
  YB_REQUIRE(d.Cin > 0 && d.Cin % 8 == 0 && d.in_cstride % 8 == 0 && d.in_cstride >= d.Cin && d.out_cstride % 8 == 0 &&
                 d.out_cstride >= d.Cout,
             "avgpool: C and the channel strides must be multiples of 8 with cstride >= C, got %d/%d/%d", d.Cin,
             d.in_cstride, d.out_cstride);
  YB_REQUIRE(d.N >= 1 && d.N <= 65535 && d.H >= 1 && d.W >= 1, "avgpool: empty or too large input (N=%d H=%d W=%d)",
             d.N, d.H, d.W);
  YB_REQUIRE(static_cast<long long>(d.H) * d.W < (1ll << 31), "avgpool: map too large");
  YB_REQUIRE(d.Ho == 1 && d.Wo == 1, "avgpool: output extent must be 1x1, got (%d,%d)", d.Ho, d.Wo);
  YB_REQUIRE(aligned16(d.in) && aligned16(d.out), "avgpool: tensors must be 16-byte aligned");
  return YB_OK;
}

int avgpool_launch(const yb_op_desc& d, cudaStream_t stream) {
  PoolParams p;
  p.in = static_cast<const uint16_t*>(d.in);
  p.out = static_cast<uint16_t*>(d.out);
  p.HW = d.H * d.W;
  p.C8 = d.Cin >> 3;
  p.in_cs = d.in_cstride, p.out_cs = d.out_cstride;
  p.octs = p.C8 < kOcts ? p.C8 : kOcts;
  p.lanes = kPoolThreads / p.octs;
  YB_CHECK_CUDA(launch_pdl(d.dtype == YB_BF16 ? avgpool_kernel<true> : avgpool_kernel<false>,
                           dim3(static_cast<unsigned>((p.C8 + p.octs - 1) / p.octs), static_cast<unsigned>(d.N)),
                           dim3(kPoolThreads), 0, stream, p));
  return YB_OK;
}

}  // namespace yb
