// FP8 (e4m3) Conv2d(+folded BN)+activation(+residual) as an implicit GEMM on the Hopper tensor cores, and the
// fp16/bf16 -> e4m3 quantisation op of FP8 plans.
//
//   acc[m, co] = sum_{r,s,ci} Xq[n, ho*stride - pad + r, wo*stride - pad + s, ci] * Wq[co, r, s, ci]     (fp32)
//   v = act(acc * m[co] + bias[co]) [+ Rq * s_res],  out = RN_satfinite(v / s_out) (e4m3) or RN(v) (fp16 / bf16)
//
// Xq = X / s_in, Wq[co] = W[co] / s_w[co] and Rq = R / s_res are e4m3; every scale is a power of two, so the multiplier
// m[co] = s_w[co] * s_in and the divisions are exact and the only roundings are the fp32 accumulation and the final
// conversion (include/yolort_b200.h, DESIGN.md "FP8 inference").
//
// Same structure as conv_wgmma_kernel (conv_sm90.cu): persistent, one CTA per SM, 128 x block_n output tiles, a TMA
// producer warp (2-D tiled rows for 1x1/s1, the 4-D im2col map for 3x3/s1 and 3x3/s2) feeding an mbarrier ring, and two
// consumer warpgroups of 64 accumulator rows each running wgmma m64nNk32 e4m3 with both operands K-major.  One byte per
// element: a 128-byte swizzled operand row holds 128 channels, and a K step of 32 channels advances the descriptors by
// the same 32 bytes as a K=16 step of the fp16 kernel.  The epilogue runs on the fragments and stores through swizzled
// shared-memory staging boxes and TMA into channel windows (out_cstride).  No chained tails, no fused decode.
#include "common.cuh"
#include "conv_sm90.h"
#include "conv_epilogue.cuh"
#include "wgmma_e4m3.cuh"

namespace yb {

namespace {

constexpr int kBlockM = 128;
constexpr int kMaxStages = 12;
constexpr int kConsumers = 2;
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kStageBufBytes = 128 * 128;   // 128 rows x 128 bytes (128 e4m3 or 64 fp16 columns)
constexpr int kStageBufs = 2;
constexpr int kMaxBlockN = 256;
constexpr size_t kSmemBudget = 216 * 1024;
constexpr uint32_t kConsumerBar = 1;

constexpr int kOutE4m3 = 0, kOutF16 = 1, kOutBf16 = 2;

struct Fp8ConvParams {
  int M, block_n, block_k;     // block_k: channels (= bytes) of one k-iteration: 128, 64 or 32
  int ksize, chunks, num_k_iters;
  int mode;                    // 0: 2-D tiled rows (1x1 stride 1), 1: 4-D im2col
  int HoWo, Wo, stride, pad;
  int stages, kpg, b_resident;
  uint32_t b_res_bytes;
  int n_tiles, num_tiles;
  int store_cols;              // columns per TMA store box
  int kk_last;                 // K=32 steps of the LAST channel chunk
  uint32_t a_stage_bytes, b_stage_bytes;
  int Cout_pad;
  const float* bias;           // [Cout_pad] bias, [Cout_pad] m[c], {s_res, 1/s_out}
  EpilogueParams ep;           // Cout, act, is_bf16 (16-bit outputs), residual (e4m3 view), res_cstride
};

__device__ __forceinline__ void consumer_sync() { named_bar_sync(kConsumerBar, 128 * kConsumers); }

// (lo, hi) -> two e4m3 bytes, lo at the lower address; round to nearest even, saturating at +-448
__device__ __forceinline__ uint16_t f32x2_to_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 e4m3x2_to_float2(uint16_t v) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(v));
  return __half22float2(*reinterpret_cast<__half2*>(&h));
}

// One TMA-store box: tile columns [c0, c0 + cols) of this thread's fragment -> staging rows of cols * esz bytes under
// the swizzle of that width (16-byte rows: none).
template <int kN, int kOut>
__device__ __forceinline__ void fp8_epilogue_box(const Fp8ConvParams& p, const float* acc, int c0, int cols,
                                                 const float* __restrict__ s_bias, const float* __restrict__ s_mul,
                                                 const FragRows& fr, int n0, float s_res, float inv_out, uint8_t* buf,
                                                 int lane) {
  constexpr int esz = kOut == kOutE4m3 ? 1 : 2;
  const int row_bytes = cols * esz;
  const int q2 = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kN / 8; ++j) {
    if (8 * j >= c0 && 8 * j < c0 + cols) {
      const int col = 8 * j + q2;
      const float b0 = s_bias[col], b1 = s_bias[col + 1];
      const float m0 = s_mul[col], m1 = s_mul[col + 1];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const float v0 = fmaf(acc[4 * j + 2 * rr], m0, b0), v1 = fmaf(acc[4 * j + 2 * rr + 1], m1, b1);
        const int r = fr.loc[rr];
        const int byte = (col - c0) * esz;
        const int chunk = row_bytes >= 32 ? swizzle_chunk(r, byte >> 4, row_bytes) : 0;
        uint8_t* dst = buf + r * row_bytes + chunk * 16 + (byte & 15);
        if constexpr (kOut == kOutE4m3) {
          float a0 = v0, a1 = v1;
          act_pair(p.ep, a0, a1);
          const int gcol = n0 + col;
          if (p.ep.residual != nullptr && fr.ok[rr] && gcol < p.ep.Cout) {   // Cout % 16 == 0: a pair never straddles it
            const uint8_t* res = static_cast<const uint8_t*>(p.ep.residual) + fr.row[rr] * p.ep.res_cstride + gcol;
            const float2 f = e4m3x2_to_float2(__ldg(reinterpret_cast<const unsigned short*>(res)));
            a0 += f.x * s_res;
            a1 += f.y * s_res;
          }
          *reinterpret_cast<uint16_t*>(dst) = f32x2_to_e4m3x2(a0 * inv_out, a1 * inv_out);
        } else {
          *reinterpret_cast<uint32_t*>(dst) = epilogue_pair<kOut == kOutBf16>(p.ep, v0, v1, fr.row[rr], fr.ok[rr], n0 + col);
        }
      }
    }
  }
}

template <int kN, int kOut>
__global__ void __launch_bounds__(kThreads, 1)
conv_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const __grid_constant__ CUtensorMap tmap_out, const Fp8ConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ __align__(8) uint64_t b_full;
  __shared__ __align__(16) float s_bias[kMaxBlockN];
  __shared__ __align__(16) float s_mul[kMaxBlockN];

  uint8_t* tiles = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const uint32_t stage_bytes = p.kpg * (p.a_stage_bytes + (p.b_resident ? 0u : p.b_stage_bytes));
  uint8_t* b_res = tiles + static_cast<size_t>(p.stages) * stage_bytes;
  uint8_t* staging = b_res + p.b_res_bytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumers);
    }
    mbar_init(&b_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // Programmatic dependent launch: resident weights do not depend on the previous kernel and stream in before the wait.
  if (threadIdx.x == 0 && p.b_resident) {
    mbar_expect_tx(&b_full, p.num_k_iters * p.block_n * p.block_k);
    for (int it = 0; it < p.num_k_iters; ++it)
      tma_load_2d(&tmap_b, &b_full, b_res + it * p.b_stage_bytes, it * p.block_k, 0);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp < 4) {
    regs_producer<1>();
    if (warp != 0) return;
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    const uint32_t a_bytes = kBlockM * p.block_k, b_bytes = p.block_n * p.block_k;
    int kit = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m_tile = tile / p.n_tiles;
      const int n0 = (tile - m_tile * p.n_tiles) * p.block_n;
      const int m0 = m_tile * kBlockM;
      int cw = 0, ch = 0, cn = 0;
      if (p.mode == 1) {
        cn = m0 / p.HoWo;
        const int rem = m0 - cn * p.HoWo;
        const int ho = rem / p.Wo;
        const int wo = rem - ho * p.Wo;
        ch = ho * p.stride - p.pad;
        cw = wo * p.stride - p.pad;
      }
      for (int it0 = 0; it0 < p.num_k_iters; it0 += p.kpg, ++kit) {
        const int cnt = min(p.kpg, p.num_k_iters - it0);
        const int s = kit % p.stages;
        const uint32_t ph = (kit / p.stages) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* a_dst = tiles + s * stage_bytes;
        uint8_t* b_dst = a_dst + p.kpg * p.a_stage_bytes;
        if (YB_ELECT()) {
          mbar_expect_tx(&full_bar[s], cnt * (a_bytes + (p.b_resident ? 0u : b_bytes)));
          for (int j = 0; j < cnt; ++j) {
            const int it = it0 + j;
            const int tap = it / p.chunks;
            const int chunk = it - tap * p.chunks;
            if (p.mode == 0) {
              tma_load_2d(&tmap_a, &full_bar[s], a_dst + j * p.a_stage_bytes, chunk * p.block_k, m0);
            } else {
              const int r = tap / p.ksize;
              const int sx = tap - r * p.ksize;
              tma_load_im2col_4d(&tmap_a, &full_bar[s], a_dst + j * p.a_stage_bytes, chunk * p.block_k, cw, ch, cn,
                                 static_cast<uint16_t>(sx), static_cast<uint16_t>(r));
            }
            if (!p.b_resident) tma_load_2d(&tmap_b, &full_bar[s], b_dst + j * p.b_stage_bytes, it * p.block_k, n0);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: MMA + epilogue of 64 rows each =====================
  regs_consumer<1>();
  const int g = (warp >> 2) - 1;
  const int wq = warp & 3;
  const bool issuer = threadIdx.x == 128;
  const int ctid = threadIdx.x - 128;
  FragRows fr;
  fr.loc[0] = g * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  const uint32_t row_bytes = p.block_k;
  const uint32_t ab_hi = desc_hi(row_bytes, 8 * row_bytes);
  const uint32_t a_half16 = (64 * row_bytes) >> 4;
  const uint32_t a_step16 = p.a_stage_bytes >> 4, b_step16 = p.b_stage_bytes >> 4;
  const uint32_t b_res_lo0 = smem_lo16(b_res);
  const int kk = p.block_k >> 5;
  const float s_res = __ldg(p.bias + 2 * p.Cout_pad), inv_out = __ldg(p.bias + 2 * p.Cout_pad + 1);
  float acc[kN / 2];

  const bool fixed_n = (gridDim.x % p.n_tiles) == 0;
  if (fixed_n) {
    const int n0f = (blockIdx.x % p.n_tiles) * p.block_n;
    for (int i = ctid; i < p.block_n; i += 128 * kConsumers) {
      const bool in = n0f + i < p.Cout_pad;
      s_bias[i] = in ? __ldg(p.bias + n0f + i) : 0.f;
      s_mul[i] = in ? __ldg(p.bias + p.Cout_pad + n0f + i) : 0.f;
    }
  }
  consumer_sync();
  if (p.b_resident) mbar_wait(&b_full, 0);

  int kit = 0, store_idx = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m_tile = tile / p.n_tiles;
    const int n0 = (tile - m_tile * p.n_tiles) * p.block_n;
    const int m0 = m_tile * kBlockM;
    if (!fixed_n) {
      consumer_sync();
      for (int i = ctid; i < p.block_n; i += 128 * kConsumers) {
        const bool in = n0 + i < p.Cout_pad;
        s_bias[i] = in ? __ldg(p.bias + n0 + i) : 0.f;
        s_mul[i] = in ? __ldg(p.bias + p.Cout_pad + n0 + i) : 0.f;
      }
    }

    int chunk = 0, prev_s = -1;
    for (int it0 = 0; it0 < p.num_k_iters; it0 += p.kpg, ++kit) {
      const int cnt = min(p.kpg, p.num_k_iters - it0);
      const int s = kit % p.stages;
      mbar_wait(&full_bar[s], (kit / p.stages) & 1);
      const uint32_t a_lo0 = smem_lo16(tiles + s * stage_bytes) + g * a_half16;
      const uint32_t b_lo0 = p.b_resident ? b_res_lo0 + it0 * b_step16 : smem_lo16(tiles + s * stage_bytes) + p.kpg * a_step16;
      wgmma_fence();
      int ch = chunk;
      for (int j = 0; j < cnt; ++j) {
        const int kc = ch == p.chunks - 1 ? p.kk_last : kk;
        for (int k = 0; k < kc; ++k)
          wgmma_e4m3<kN>(acc, desc_lohi(a_lo0 + j * a_step16 + 2 * k, ab_hi), desc_lohi(b_lo0 + j * b_step16 + 2 * k, ab_hi),
                         (it0 | j | k) != 0 ? 1u : 0u);
        if (++ch == p.chunks) ch = 0;
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_s >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
      chunk = ch;
    }
    wgmma_wait<0>();
    fence_acc<kN / 2>(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_s]);
    if (!fixed_n) consumer_sync();

    fr.row[0] = static_cast<long long>(m0) + fr.loc[0];
    fr.row[1] = static_cast<long long>(m0) + fr.loc[1];
    fr.ok[0] = fr.row[0] < p.M;
    fr.ok[1] = fr.row[1] < p.M;
    for (int c0 = 0; c0 < kN; c0 += p.store_cols, ++store_idx) {
      // two staging buffers: the issuer waits until the previous store has read the buffer the next box overwrites
      uint8_t* buf = staging + (store_idx & 1) * kStageBufBytes;
      fp8_epilogue_box<kN, kOut>(p, acc, c0, p.store_cols, s_bias, s_mul, fr, n0, s_res, inv_out, buf, lane);
      fence_proxy_async_smem();
      if (issuer) tma_store_wait_read<0>();
      consumer_sync();
      if (issuer) {
        if (n0 + c0 < p.ep.Cout) tma_store_2d(&tmap_out, buf, n0 + c0, m0);
        tma_store_commit();
      }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

// 16 channels (two 16-byte loads of fp16 / bf16, one 16-byte store of e4m3) per thread
template <bool kBf16>
__global__ void quantize_e4m3_kernel(const uint16_t* __restrict__ in, int in_cs, uint8_t* __restrict__ out, int out_cs,
                                     long long pixels, int C, const float* __restrict__ inv_scale) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c16n = C >> 4;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= pixels * c16n) return;
  const int c16 = static_cast<int>(idx % c16n);
  const long long pix = idx / c16n;
  const uint4* src = reinterpret_cast<const uint4*>(in + pix * in_cs + c16 * 16);
  const uint4 v[2] = {__ldg(src), __ldg(src + 1)};
  const float s = __ldg(inv_scale);
  uint32_t w[4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t u[4] = {v[h].x, v[h].y, v[h].z, v[h].w};
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float2 a = unpack2<kBf16>(u[2 * q]), b = unpack2<kBf16>(u[2 * q + 1]);
      w[2 * h + q] = static_cast<uint32_t>(f32x2_to_e4m3x2(a.x * s, a.y * s)) |
                     (static_cast<uint32_t>(f32x2_to_e4m3x2(b.x * s, b.y * s)) << 16);
    }
  }
  *reinterpret_cast<uint4*>(out + pix * out_cs + c16 * 16) = make_uint4(w[0], w[1], w[2], w[3]);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

using Fp8KernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const Fp8ConvParams);

template <int kOut>
Fp8KernelFn select_fp8_kernel_t(int block_n) {
  switch (block_n) {
    case 16: return conv_fp8_kernel<16, kOut>;
    case 32: return conv_fp8_kernel<32, kOut>;
    case 64: return conv_fp8_kernel<64, kOut>;
    case 128: return conv_fp8_kernel<128, kOut>;
    default: return conv_fp8_kernel<256, kOut>;
  }
}

int out_kind(const yb_op_desc& d) {
  return (d.reserved & YB_CONV_E4M3_F16_OUT) ? kOutF16 : ((d.reserved & YB_CONV_E4M3_BF16_OUT) ? kOutBf16 : kOutE4m3);
}

// Pure host logic: validation, tiling, pipeline depth and launch shape (no driver calls).
int fp8_configure(const yb_op_desc& d, Fp8ConvParams& kp, dim3& grid, size_t& smem_bytes) {
  YB_REQUIRE(d.dtype == YB_F8E4M3, "e4m3 conv: dtype must be YB_F8E4M3");
  constexpr int kOutBits = YB_CONV_E4M3_F16_OUT | YB_CONV_E4M3_BF16_OUT;
  YB_REQUIRE((d.reserved & ~kOutBits) == 0 && (d.reserved & kOutBits) != kOutBits,
             "e4m3 conv: reserved may only set bit 4 (fp16 output) or bit 5 (bf16 output), got 0x%x", d.reserved);
  YB_REQUIRE(d.decode == nullptr && d.chain == nullptr, "e4m3 conv: no fused decode and no chained tail");
  YB_REQUIRE(d.act >= YB_ACT_NONE && d.act <= YB_ACT_RELU, "e4m3 conv: unknown activation %d", d.act);
  YB_REQUIRE((d.ksize == 1 && d.stride == 1 && d.pad == 0) || (d.ksize == 3 && d.pad == 1 && (d.stride == 1 || d.stride == 2)),
             "e4m3 conv: 1x1/s1/p0, 3x3/s1/p1 or 3x3/s2/p1, got %dx%d/s%d/p%d", d.ksize, d.ksize, d.stride, d.pad);
  const int out = out_kind(d);
  const int oq = out == kOutE4m3 ? 16 : 8;   // 16-byte windows
  YB_REQUIRE(d.Cin % 16 == 0 && d.in_cstride % 16 == 0 && d.in_cstride >= d.Cin,
             "e4m3 conv: Cin/in_cstride must be multiples of 16, got %d/%d", d.Cin, d.in_cstride);
  YB_REQUIRE(d.Cout % oq == 0 && d.out_cstride % oq == 0 && d.out_cstride >= d.Cout,
             "e4m3 conv: Cout/out_cstride must be multiples of %d, got %d/%d", oq, d.Cout, d.out_cstride);
  YB_REQUIRE(d.Cin_pad % 32 == 0 && d.Cin_pad >= d.Cin, "e4m3 conv: Cin_pad must be a multiple of 32 >= Cin");
  YB_REQUIRE(d.Cout_pad % 16 == 0 && d.Cout_pad >= d.Cout, "e4m3 conv: Cout_pad must be a multiple of 16 >= Cout");
  YB_REQUIRE(aligned16(d.in) && aligned16(d.out) && aligned16(d.weight) && (reinterpret_cast<uintptr_t>(d.bias) & 3) == 0,
             "e4m3 conv: in, out and weight must be 16-byte aligned, bias 4-byte aligned");
  YB_REQUIRE(d.residual == nullptr || (out == kOutE4m3 && aligned16(d.residual) && d.res_cstride % 16 == 0 &&
                                       d.res_cstride >= d.Cout),
             "e4m3 conv: a residual needs the e4m3 output, 16-byte alignment and res_cstride a multiple of 16");
  kp = Fp8ConvParams();
  const int rc = conv_rows(d, "e4m3 conv", &kp.M);
  if (rc != YB_OK) return rc;
  const int m_tiles = (kp.M + kBlockM - 1) / kBlockM;
  const int block_n = conv_block_n(d.Cout, m_tiles, false);
  const int n_tiles = (d.Cout + block_n - 1) / block_n;
  kp.block_n = block_n;
  kp.n_tiles = n_tiles;
  kp.num_tiles = m_tiles * n_tiles;
  kp.block_k = (d.Cin_pad % 128 == 0) ? 128 : ((d.Cin_pad % 64 == 0) ? 64 : 32);
  kp.ksize = d.ksize;
  kp.chunks = d.Cin_pad / kp.block_k;
  kp.num_k_iters = d.ksize * d.ksize * kp.chunks;
  kp.mode = d.ksize == 1 ? 0 : 1;
  kp.HoWo = d.Ho * d.Wo;
  kp.Wo = d.Wo;
  kp.stride = d.stride;
  kp.pad = d.pad;
  // store boxes of 128-byte rows where the tile allows (e4m3: up to 128 columns, 16-bit outputs: up to 64)
  const int max_cols = out == kOutE4m3 ? 128 : 64;
  kp.store_cols = block_n < max_cols ? block_n : max_cols;
  kp.kk_last = (d.Cin - (kp.chunks - 1) * kp.block_k + 31) / 32;
  if (kp.kk_last < 1) kp.kk_last = 1;
  if (kp.kk_last > (kp.block_k >> 5)) kp.kk_last = kp.block_k >> 5;
  kp.a_stage_bytes = kBlockM * kp.block_k;
  kp.b_stage_bytes = (static_cast<uint32_t>(kp.block_n * kp.block_k) + 1023u) & ~1023u;
  kp.Cout_pad = d.Cout_pad;
  kp.bias = d.bias;
  kp.ep.Cout = d.Cout;
  kp.ep.act = d.act;
  kp.ep.is_bf16 = out == kOutBf16;
  kp.ep.residual = d.residual;
  kp.ep.res_cstride = d.res_cstride;

  KPipeline pipe;
  const int prc = size_k_pipeline(kSmemBudget, static_cast<size_t>(kStageBufs) * kStageBufBytes + 1024, kp.a_stage_bytes,
                                  kp.b_stage_bytes, kp.num_k_iters, n_tiles == 1, kMaxStages, "e4m3 conv", kp.block_n, &pipe);
  if (prc != YB_OK) return prc;
  kp.b_resident = pipe.b_resident;
  kp.b_res_bytes = pipe.b_res_bytes;
  kp.kpg = pipe.kpg;
  kp.stages = pipe.stages;
  grid = dim3(kp.num_tiles < num_sms() ? kp.num_tiles : num_sms(), 1, 1);
  smem_bytes = pipe.smem;
  return YB_OK;
}

}  // namespace

int fp8_conv_config(const yb_op_desc& d, yb_conv_info* info) {
  Fp8ConvParams kp;
  dim3 grid;
  size_t smem = 0;
  const int rc = fp8_configure(d, kp, grid, smem);
  if (rc == YB_OK && info) {   // yb_conv_config: see include/yolort_b200.h
    info->kernel = YB_CONV_KERNEL_E4M3;
    info->block_n = kp.block_n;
    info->n_tiles = kp.n_tiles;
    info->weights_resident = kp.b_resident;
    info->tiles_per_pass = 1;
    info->slots = kp.stages;
    info->ring = kp.kpg;
    info->store_cols = kp.store_cols;
    info->store_bufs = kStageBufs;
    info->groups = kConsumers;
    info->resident_ctas = 1;
    info->smem_bytes = static_cast<int>(smem);
    info->grid = static_cast<int>(grid.x);
    info->tiling = YB_CONV_TILING_ROWS;
    info->m_tiles = kp.num_tiles / kp.n_tiles;
    info->work_items = kp.num_tiles;
  }
  return rc;
}

struct Fp8ConvOp final : ConvOp {
  CUtensorMap tmap_a, tmap_b, tmap_out;
  Fp8ConvParams kp;
  Fp8KernelFn fn = nullptr;
  dim3 grid;
  size_t smem_bytes;
  int launch(cudaStream_t stream) const override {
    YB_CHECK_CUDA(launch_pdl(fn, grid, dim3(kThreads), smem_bytes, stream, tmap_a, tmap_b, tmap_out, kp));
    return YB_OK;
  }
};

int fp8_conv_create(const yb_op_desc& d, ConvOp** out) {
  Fp8ConvOp* op = new Fp8ConvOp();
  const Fp8ConvParams& kp = op->kp;
  int rc = fp8_configure(d, op->kp, op->grid, op->smem_bytes);   // validates before any driver call
  const CUtensorMapDataType u8 = CU_TENSOR_MAP_DATA_TYPE_UINT8;
  if (rc == YB_OK)
    rc = kp.mode == 0 ? tmap_matrix(&op->tmap_a, "e4m3 conv input", u8, d.in, d.Cin, kp.M, d.in_cstride, kp.block_k, kBlockM,
                                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B)
                      : tmap_im2col(&op->tmap_a, "e4m3 conv input", u8, d, kp.block_k, kBlockM);
  const int ktot = d.ksize * d.ksize * d.Cin_pad;
  if (rc == YB_OK)
    rc = tmap_matrix(&op->tmap_b, "e4m3 conv weights", u8, d.weight, ktot, d.Cout_pad, ktot, kp.block_k, kp.block_n,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  const int ok = out_kind(d);
  const CUtensorMapDataType dt = ok == kOutE4m3 ? u8 : (ok == kOutBf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                                       : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  if (rc == YB_OK)
    rc = tmap_matrix(&op->tmap_out, "e4m3 conv output", dt, d.out, d.Cout, kp.M, d.out_cstride, kp.store_cols, kBlockM,
                     CU_TENSOR_MAP_L2_PROMOTION_NONE);
  if (rc == YB_OK) {
    op->fn = ok == kOutE4m3 ? select_fp8_kernel_t<kOutE4m3>(kp.block_n)
                            : (ok == kOutF16 ? select_fp8_kernel_t<kOutF16>(kp.block_n)
                                               : select_fp8_kernel_t<kOutBf16>(kp.block_n));
    const cudaError_t e = cudaFuncSetAttribute(op->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBudget));
    if (e != cudaSuccess) {
      set_error("e4m3 conv: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      rc = YB_ERR_CUDA;
    }
  }
  if (rc != YB_OK) {
    delete op;
    return rc;
  }
  *out = op;
  return YB_OK;
}

int quantize_configure_check(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "quantize: dtype (the source type) must be f16 or bf16");
  YB_REQUIRE(d.Cin == d.Cout && d.Cin > 0 && d.Cin % 16 == 0, "quantize: Cin == Cout, a multiple of 16, got %d/%d", d.Cin,
             d.Cout);
  YB_REQUIRE(d.in_cstride % 8 == 0 && d.in_cstride >= d.Cin && d.out_cstride % 16 == 0 && d.out_cstride >= d.Cout,
             "quantize: in_cstride must be a multiple of 8, out_cstride of 16");
  YB_REQUIRE(d.Ho == d.H && d.Wo == d.W && d.N > 0 && d.H > 0 && d.W > 0, "quantize: the output has the input's extent");
  YB_REQUIRE(aligned16(d.in) && aligned16(d.out) && d.bias != nullptr && (reinterpret_cast<uintptr_t>(d.bias) & 3) == 0,
             "quantize: in and out must be 16-byte aligned and bias (1/s) set");
  YB_REQUIRE(d.weight == nullptr && d.residual == nullptr && d.decode == nullptr && d.chain == nullptr && d.act == 0 &&
                 d.reserved == 0,
             "quantize: weight, residual, decode and chain must be NULL, act and reserved 0");
  return YB_OK;
}

int quantize_launch(const yb_op_desc& d, cudaStream_t stream) {
  const long long pixels = static_cast<long long>(d.N) * d.H * d.W;
  const long long total = pixels * (d.Cin >> 4);
  const dim3 grid(static_cast<unsigned>((total + 255) / 256));
  const uint16_t* in = static_cast<const uint16_t*>(d.in);
  uint8_t* out = static_cast<uint8_t*>(d.out);
  YB_CHECK_CUDA(launch_pdl(d.dtype == YB_BF16 ? quantize_e4m3_kernel<true> : quantize_e4m3_kernel<false>, grid, dim3(256), 0,
                           stream, in, d.in_cstride, out, d.out_cstride, pixels, d.Cin, d.bias));
  return YB_OK;
}

}  // namespace yb
