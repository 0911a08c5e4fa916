// Epilogue helpers shared by the convolution kernels (bias + activation + residual + pack, swizzled staging).
//
// The accumulator of a 128-row tile lives in the registers of the two consumer warpgroups, 64 rows each, in the wgmma
// fragment layout: thread t of warpgroup g (warp w = t / 32, lane l) holds, for every 8-column block j,
//   acc[4j + 0..1] = row g*64 + 16w + l/4,     columns 8j + 2(l%4) + 0..1
//   acc[4j + 2..3] = row g*64 + 16w + l/4 + 8, same columns.
// Each thread turns its column pairs into packed fp16/bf16 pairs and writes them into the swizzled staging box that a
// TMA store (and, for a chained tail, a wgmma operand descriptor) reads.
#pragma once
#include "common.cuh"

namespace yb {

// fields of the kernel parameter block the epilogue needs
struct EpilogueParams {
  int Cout;
  int act, is_bf16;
  const void* residual;
  int res_cstride;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// SiLU(v) = v / (1 + 2^(-v*log2 e)) in fp32; both transcendental steps on the MUFU pipe.
__device__ __forceinline__ float silu(float v) { return v * rcp_approx(1.0f + ex2_approx(v * -1.4426950408889634f)); }

template <bool kBf16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (kBf16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
template <bool kBf16>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
  if constexpr (kBf16) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  } else {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
}

// Physical 16-byte chunk index of logical chunk `j` in row `r` of a tile whose rows are `row_bytes`
// long, under the TMA/wgmma swizzle of the same width (address bits [4,7) ^= bits [7,10), truncated).
__device__ __forceinline__ int swizzle_chunk(int r, int j, int row_bytes) {
  if (row_bytes == 128) return j ^ (r & 7);
  if (row_bytes == 64) return j ^ ((r >> 1) & 3);
  return j ^ ((r >> 2) & 1);
}

// The two accumulator rows of this thread: position in the tile, output pixel, and whether it exists.
struct FragRows {
  int loc[2];
  long long row[2];
  bool ok[2];
};

// bias -> activation (SiLU / linear, or the r3.1 Hardswish / LeakyReLU(0.1)) -> + shortcut, in fp32
template <bool kBf16>
__device__ __forceinline__ uint32_t epilogue_pair(const EpilogueParams& p, float v0, float v1, long long row, bool row_ok,
                                                  int gcol) {
  if (p.act == YB_ACT_SILU) {
    v0 = silu(v0);
    v1 = silu(v1);
  } else if (p.act == YB_ACT_HARDSWISH) {
    v0 = v0 * fminf(fmaxf(v0 + 3.0f, 0.f), 6.0f) * (1.0f / 6.0f);
    v1 = v1 * fminf(fmaxf(v1 + 3.0f, 0.f), 6.0f) * (1.0f / 6.0f);
  } else if (p.act == YB_ACT_LEAKY01) {
    v0 = v0 > 0.f ? v0 : v0 * 0.1f;
    v1 = v1 > 0.f ? v1 : v1 * 0.1f;
  }
  if (p.residual != nullptr && row_ok && gcol < p.Cout) {   // Cout % 8 == 0: a pair never straddles it
    const uint16_t* r = reinterpret_cast<const uint16_t*>(p.residual) + row * p.res_cstride + gcol;
    const float2 f = unpack2<kBf16>(__ldg(reinterpret_cast<const unsigned int*>(r)));
    v0 += f.x;
    v1 += f.y;
  }
  return pack2<kBf16>(v0, v1);
}

// One TMA-store box: tile columns [c0, c0 + cols) of this thread's fragment -> swizzled staging rows of `cols * 2`
// bytes.  kN: the accumulator columns `acc` holds (the loop over 8-column blocks is unrolled so that every register
// index is a constant).  n0: output channel of tile column 0; s_bias is indexed by tile column.
template <bool kBf16, int kN>
__device__ __forceinline__ void epilogue_box(const EpilogueParams& p, const float* acc, int c0, int cols,
                                             const float* __restrict__ s_bias, const FragRows& fr, int n0, uint8_t* buf,
                                             int lane) {
  const int row_bytes = cols * 2;
  const int q2 = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kN / 8; ++j) {
    if (8 * j >= c0 && 8 * j < c0 + cols) {
      const int col = 8 * j + q2;
      const float b0 = s_bias[col], b1 = s_bias[col + 1];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const uint32_t o = epilogue_pair<kBf16>(p, acc[4 * j + 2 * rr] + b0, acc[4 * j + 2 * rr + 1] + b1,
                                                fr.row[rr], fr.ok[rr], n0 + col);
        const int r = fr.loc[rr];
        *reinterpret_cast<uint32_t*>(buf + r * row_bytes + swizzle_chunk(r, (col - c0) >> 3, row_bytes) * 16 +
                                     ((col - c0) & 7) * 2) = o;
      }
    }
  }
}

}  // namespace yb
