// Conv2d(+folded BN)+SiLU(+residual) as an implicit GEMM on the Hopper tensor cores (wgmma).
//
//   D[m, co] = sum_{r,s,ci} X[n, ho*stride - pad + r, wo*stride - pad + s, ci] * W[co, r, s, ci]
//   m = (n*Ho + ho)*Wo + wo      (NHWC activations, K-major weights)
//
// Replaces the arithmetic of yolort/v5/models/common.py:42-73 (Conv = conv2d -> BN(eps 1e-3) -> SiLU),
// :94-116 (Bottleneck residual) and the 1x1 head convs of yolort/models/box_head.py:35-37,68-82.
//
// Persistent kernel, one CTA per SM, static round-robin over 128 x block_n output tiles, 384 threads:
//   warpgroup 0 (producer, 40 registers): warp 0 issues the TMA loads.  A tiles come from a 4-D im2col tensor map (the
//                TMA engine walks 128 output pixels, applies padding/stride and zero-fills the halo) or, for 1x1/s1
//                convs, from a 2-D tiled map; B tiles (weights) from a 2-D tiled map.  Both land in shared memory in the
//                32/64/128-byte swizzled K-major layout wgmma reads.  The producer runs ahead across tile boundaries.
//   warpgroups 1-2 (consumers, 232 registers): each multiplies 64 rows of the tile (wgmma m64nNk16, N = block_n, fp32
//                accumulators in registers), then runs the epilogue on its fragment: +bias -> activation -> (+residual)
//                -> fp16/bf16 -> swizzled shared-memory staging -> TMA store into the NHWC destination view (a channel
//                window of a concat buffer is just a strided tensor map; ragged M is clipped by the TMA unit).
// The kernel is a template over (dtype, activation family, fused decode, chained tail).  A chained tail
// (conv_chain.cuh) is a second, pointwise GEMM over the tile the epilogue has just staged: the consumers multiply the
// staged boxes with the resident tail weights and a second epilogue pass stores the result.
#include <cstdlib>

#include "common.cuh"
#include "conv_sm90.h"
#include "conv_epilogue.cuh"
#include "conv_chain.cuh"
#include "decode_common.cuh"

namespace yb {

namespace {

constexpr int kBlockM = 128;
constexpr int kMaxStages = 12;
constexpr int kConsumers = 2;                         // consumer warpgroups (64 accumulator rows each)
constexpr int kThreads = 128 * (1 + kConsumers);
constexpr int kStageBufBytes = 128 * 128;  // 128 rows x (up to) 64 columns x 2 B
constexpr int kStageBufs = 2;              // staging boxes, shared by the two consumer warpgroups
constexpr int kMaxBlockN = 256;
constexpr size_t kSmemBudget = 216 * 1024;  // dynamic shared memory per CTA (227 KB limit minus static)
constexpr uint32_t kConsumerBar = 1;        // named barrier of the 256 consumer threads

struct ConvKernelParams {
  int M, block_n, block_k;
  int ksize, chunks, num_k_iters;
  int mode;  // 0: 2-D tiled rows (1x1 stride 1), 1: 4-D im2col
  int HoWo, Wo, stride, pad;
  int stages;
  int kpg;         // k-iterations (A/B sub-tiles) carried by one pipeline stage
  int b_resident;  // weights of the (single) N tile stay in shared memory for the CTA's lifetime
  uint32_t b_res_bytes;
  int n_tiles, num_tiles;
  int store_cols;  // columns per TMA store box: 64 / 32 / 16
  int bias_len;    // length of the (padded) bias vector
  int kk_last;     // K=16 steps of the LAST channel chunk (Cin need not fill it: TMA zero-fills, the MMA skips)
  uint32_t a_stage_bytes, b_stage_bytes;
  const float* bias;
  EpilogueParams ep;
  ChainParams ch;  // chained pointwise tail (kChain kernels)
  int decode_on;        // detection head with the fused decode epilogue (no logits are stored)
  int dec_H, dec_W;     // level extent (output pixels)
  yb_head_decode dec;   // copied from the op descriptor
};

__device__ __forceinline__ void consumer_sync() { named_bar_sync(kConsumerBar, 128 * kConsumers); }

// Fused post-processing front end (yolort/models/box_head.py:328-360,418) on the head's accumulator fragment.  Objectness
// and box logits of every (row, anchor) go through a small shared-memory table (they sit in other lanes' registers);
// each thread then tests the class columns it holds and emits candidates straight into the NMS arena.
template <int kN>
__device__ __forceinline__ void decode_fragment(const yb_head_decode& D, const float* acc, const float* s_bias,
                                                const FragRows& fr, int dec_H, int dec_W, float* head, uint32_t wg_bar,
                                                int lane) {
  constexpr int kMaxA = 4;
  const int K = D.n_classes + 5;
  const int q2 = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kN / 8; ++j) {
    {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int col = 8 * j + q2 + (i & 1);
        const int a = col / K, r = col - a * K;
        if (a < D.n_anchors && r < 5) head[fr.loc[i >> 1] * 20 + a * 5 + r] = acc[4 * j + i] + s_bias[col];
      }
    }
  }
  named_bar_sync(wg_bar, 128);
  float obj[2][kMaxA];
  bool pass[2][kMaxA];
  uint32_t emitted[2] = {0u, 0u};
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
    for (int a = 0; a < kMaxA; ++a) {
      obj[rr][a] = a < D.n_anchors ? sigmoidf_ref(head[fr.loc[rr] * 20 + a * 5 + 4]) : 0.f;
      pass[rr][a] = a < D.n_anchors && fr.ok[rr] && obj[rr][a] > D.score_thresh;
    }
  }
  int n_img[2], py[2], px[2];
  const int hw = dec_H * dec_W;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    n_img[rr] = static_cast<int>(fr.row[rr] / hw);
    const int rem = static_cast<int>(fr.row[rr] - static_cast<long long>(n_img[rr]) * hw);
    py[rr] = rem / dec_W;
    px[rr] = rem - py[rr] * dec_W;
  }
  const bool any_pass = pass[0][0] || pass[0][1] || pass[0][2] || pass[0][3] || pass[1][0] || pass[1][1] ||
                        pass[1][2] || pass[1][3];
  if (any_pass) {
#pragma unroll
    for (int j = 0; j < kN / 8; ++j) {
      {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rr = i >> 1;
          const int col = 8 * j + q2 + (i & 1);
          const int a = col / K, r = col - a * K;
          const bool pa = a == 0 ? pass[rr][0] : (a == 1 ? pass[rr][1] : (a == 2 ? pass[rr][2] : (a == 3 && pass[rr][3])));
          if (pa && r >= 5) {
            const float oa = a == 0 ? obj[rr][0] : (a == 1 ? obj[rr][1] : (a == 2 ? obj[rr][2] : obj[rr][3]));
            const float score = __fmul_rn(sigmoidf_ref(acc[4 * j + i] + s_bias[col]), oa);
            if (score > D.score_thresh) {
              const int anchor_flat = D.level_start + (a * dec_H + py[rr]) * dec_W + px[rr];
              emit_candidate(D.keys, D.img_count, D.cap_per_image, n_img[rr], anchor_flat, D.n_classes, r - 5, score);
              emitted[rr] |= 1u << a;
            }
          }
        }
      }
    }
  }
  // the four lanes of a quad share their rows: one of them writes the boxes of the anchors any of them emitted
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    emitted[rr] |= __shfl_xor_sync(0xffffffffu, emitted[rr], 1);
    emitted[rr] |= __shfl_xor_sync(0xffffffffu, emitted[rr], 2);
    if ((lane & 3) == 0 && emitted[rr]) {
      const float* h = head + fr.loc[rr] * 20;
      for (int a = 0; a < D.n_anchors; ++a) {
        if (!((emitted[rr] >> a) & 1u)) continue;
        const int anchor_flat = D.level_start + (a * dec_H + py[rr]) * dec_W + px[rr];
        const float4 b = decode_box(sigmoidf_ref(h[a * 5 + 0]), sigmoidf_ref(h[a * 5 + 1]), sigmoidf_ref(h[a * 5 + 2]),
                                    sigmoidf_ref(h[a * 5 + 3]), px[rr], py[rr], D.stride_px, D.anchors_px[2 * a],
                                    D.anchors_px[2 * a + 1]);
        reinterpret_cast<float4*>(D.boxes)[static_cast<long long>(n_img[rr]) * D.anchors_per_image + anchor_flat] = b;
        atomicMax(&D.img_maxc[n_img[rr]], float_to_ordered_int(fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w))));
      }
    }
  }
  named_bar_sync(wg_bar, 128);   // the table is rewritten by the next tile
}

// kN: the wgmma N of the tile (= block_n; kN / 2 accumulator registers per thread).  kDecode: detection head with the
// fused decode (nothing stored).  kN2 != 0: a
// pointwise tail is chained onto every tile (conv_chain.cuh).
template <bool kBf16, int kN, bool kDecode, int kN2>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_w2,
                  const __grid_constant__ CUtensorMap tmap_out2, const ConvKernelParams p) {
  constexpr bool kChain = kN2 != 0;
  constexpr int kAcc = (kN > kN2 ? kN : kN2) / 2;   // accumulator registers per thread
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ __align__(8) uint64_t b_full;
  __shared__ __align__(8) uint64_t w2_full;
  __shared__ __align__(16) float s_bias[kMaxBlockN];
  __shared__ __align__(16) float s_bias2[kChain ? kMaxBlockN : 4];

  // Swizzled tiles need 1024-byte alignment.
  uint8_t* tiles = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  // stage = kpg A sub-tiles followed (unless the weights are resident) by kpg B sub-tiles
  const uint32_t stage_bytes = p.kpg * (p.a_stage_bytes + (p.b_resident ? 0u : p.b_stage_bytes));
  uint8_t* b_res = tiles + static_cast<size_t>(p.stages) * stage_bytes;   // resident weights (optional)
  uint8_t* staging = b_res + p.b_res_bytes;                                // [kStageBufs][kStageBufBytes]
  uint8_t* w2_res = staging + kStageBufs * kStageBufBytes;                 // chain: resident tail weights

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumers);   // one arrival per consumer warpgroup
    }
    mbar_init(&b_full, 1);
    mbar_init(&w2_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // Programmatic dependent launch: everything above overlapped the tail of the previous kernel in the stream.
  // Resident weights do not depend on the previous kernel: their loads are issued BEFORE the grid-dependency wait
  // and stream in while the previous kernel drains.
  if (threadIdx.x == 0 && p.b_resident) {
    const uint32_t b_bytes = p.block_n * p.block_k * 2;
    mbar_expect_tx(&b_full, p.num_k_iters * b_bytes);
    for (int it = 0; it < p.num_k_iters; ++it)
      tma_load_2d(&tmap_b, &b_full, b_res + it * p.b_stage_bytes, it * p.block_k, 0);
  }
  if constexpr (kChain) {
    if (threadIdx.x == 0) {   // tail weights: [n2][kc] chunks, resident for the CTA's lifetime
      tma_prefetch_desc(&tmap_w2);
      tma_prefetch_desc(&tmap_out2);
      mbar_expect_tx(&w2_full, p.ch.w2_chunks * p.ch.n2 * p.ch.w2_row_bytes);
      for (int j = 0; j < p.ch.w2_chunks; ++j)
        tma_load_2d(&tmap_w2, &w2_full, w2_res + j * p.ch.w2_sub_bytes, j * (p.ch.w2_row_bytes >> 1), 0);
    }
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp < 4) {
    regs_producer();
    if (warp != 0) return;
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    const uint32_t a_bytes = kBlockM * p.block_k * 2, b_bytes = p.block_n * p.block_k * 2;
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
  regs_consumer();
  const int g = (warp >> 2) - 1;
  const int wq = warp & 3;
  const bool issuer = threadIdx.x == 128;
  const int ctid = threadIdx.x - 128;
  FragRows fr;
  fr.loc[0] = g * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  const uint32_t row_bytes = p.block_k * 2;
  const uint32_t ab_hi = desc_hi(row_bytes, 8 * row_bytes);
  const uint32_t a_half16 = (64 * row_bytes) >> 4;   // this warpgroup's 64 rows of an A sub-tile
  const uint32_t a_step16 = p.a_stage_bytes >> 4, b_step16 = p.b_stage_bytes >> 4;
  const uint32_t b_res_lo0 = smem_lo16(b_res);
  const int kk = p.block_k >> 4;
  constexpr int bn = kN;
  const int store_cols = p.store_cols;
  float acc[kAcc];

  if constexpr (kChain) {   // the tail has a single N tile: its bias is the same for every tile
    for (int i = ctid; i < p.ch.n2; i += 128 * kConsumers) s_bias2[i] = (i < p.ch.bias2_len) ? __ldg(p.ch.bias2 + i) : 0.f;
  }
  // Every tile of this CTA has the same N tile when the grid is a multiple of the N-tile count (always with one N
  // tile): the bias is then loaded ONCE instead of per tile.
  const bool fixed_n = (gridDim.x % p.n_tiles) == 0;
  if (fixed_n) {
    const int n0f = (blockIdx.x % p.n_tiles) * p.block_n;
    for (int i = ctid; i < p.block_n; i += 128 * kConsumers) s_bias[i] = (n0f + i < p.bias_len) ? __ldg(p.bias + n0f + i) : 0.f;
  }
  consumer_sync();
  if (p.b_resident) mbar_wait(&b_full, 0);
  if constexpr (kChain) mbar_wait(&w2_full, 0);

  int kit = 0, store_idx = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m_tile = tile / p.n_tiles;
    const int n0 = (tile - m_tile * p.n_tiles) * p.block_n;
    const int m0 = m_tile * kBlockM;
    if (!fixed_n) {   // the previous tile's epilogue has finished with the bias (and the staging boxes)
      consumer_sync();
      for (int i = ctid; i < p.block_n; i += 128 * kConsumers) s_bias[i] = (n0 + i < p.bias_len) ? __ldg(p.bias + n0 + i) : 0.f;
    }

    // ---- main loop: stage s is released once the MMAs that read it have completed (one stage in flight) ----
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
          wgmma_mma<kBf16, kN>(acc, desc_lohi(a_lo0 + j * a_step16 + 2 * k, ab_hi), desc_lohi(b_lo0 + j * b_step16 + 2 * k, ab_hi),
                            (it0 | j | k) != 0);
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
    if (!fixed_n) consumer_sync();   // bias visible

    fr.row[0] = static_cast<long long>(m0) + fr.loc[0];
    fr.row[1] = static_cast<long long>(m0) + fr.loc[1];
    fr.ok[0] = fr.row[0] < p.M;
    fr.ok[1] = fr.row[1] < p.M;
    if constexpr (kDecode) {
      decode_fragment<kN>(p.dec, acc, s_bias, fr, p.dec_H, p.dec_W, reinterpret_cast<float*>(staging), 2 + g, lane);
    } else {
    if constexpr (kChain) {
      // chain tiles index the staging buffers by box (box b of the tile stays in buffer b until the tail GEMM has read
      // it), so the previous tile's stores must have drained both buffers before this tile writes them
      if (issuer) tma_store_wait_read<0>();
      consumer_sync();
    }
    for (int c0 = 0; c0 < bn; c0 += store_cols, ++store_idx) {
      // Two staging buffers, one barrier per box: before the barrier below the issuer waits until the PREVIOUS
      // store has finished reading its buffer, which is the one the next box will overwrite.
      uint8_t* buf = staging + (kChain ? (c0 / store_cols) : (store_idx & 1)) * kStageBufBytes;
      epilogue_box<kBf16, kN>(p.ep, acc, c0, store_cols, s_bias, fr, n0, buf, lane);
      fence_proxy_async_smem();
      if constexpr (!kChain) {
        if (issuer) tma_store_wait_read<0>();
      }
      consumer_sync();
      if (issuer) {
        if ((!kChain || p.ch.store_first) && n0 + c0 < p.ep.Cout) tma_store_2d(&tmap_out, buf, n0 + c0, m0);
        tma_store_commit();
      }
    }
    if constexpr (kChain) {
      // every box of the tile is in shared memory and visible to the async proxy (fence + barrier above)
      const uint32_t a2_hi = desc_hi(p.ch.own_row_bytes, 8 * p.ch.own_row_bytes);
      const uint32_t w2_hi = desc_hi(p.ch.w2_row_bytes, 8 * p.ch.w2_row_bytes);
      const uint32_t stag_lo = smem_lo16(staging) + ((64 * g * p.ch.own_row_bytes) >> 4);
      const uint32_t w2_lo0 = smem_lo16(w2_res);
      wgmma_fence();
      for (int j = 0; j < p.ch.own_chunks; ++j)
        for (int k = 0; k < p.ch.ksteps; ++k)
          wgmma_mma<kBf16, kChain ? kN2 : 16>(acc, desc_lohi(stag_lo + j * (kStageBufBytes >> 4) + 2 * k, a2_hi),
                            desc_lohi(w2_lo0 + j * (p.ch.w2_sub_bytes >> 4) + 2 * k, w2_hi), (j | k) != 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc<kChain ? kN2 / 2 : 8>(acc);
      // the tail's boxes reuse the staging buffers: the operand boxes are dead (both warpgroups' tail GEMMs have
      // completed), but the stores of the first output may still be reading them
      if (issuer) tma_store_wait_read<0>();
      consumer_sync();
      const int s2 = chain_store2_cols(p.ch.n2);
      for (int c0 = 0; c0 < p.ch.n2; c0 += s2) {
        uint8_t* buf = staging + ((c0 / s2) & 1) * kStageBufBytes;
        epilogue_box<kBf16, kChain ? kN2 : 16>(p.ch.ep2, acc, c0, s2, s_bias2, fr, 0, buf, lane);
        fence_proxy_async_smem();
        if (issuer) tma_store_wait_read<0>();   // box k + 1 overwrites the buffer of box k - 1
        consumer_sync();
        if (issuer) {
          if (c0 < p.ch.ep2.Cout) tma_store_2d(&tmap_out2, buf, c0, m0);
          tma_store_commit();
        }
      }
    }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

// ---- host side -----------------------------------------------------------------------------------
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const int*, const int*,
                                   cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

EncodeTiledFn g_encode_tiled = nullptr;
EncodeIm2colFn g_encode_im2col = nullptr;

int load_driver_entry_points() {
  if (g_encode_tiled && g_encode_im2col) return YB_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  YB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  YB_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess,
             "cuTensorMapEncodeTiled not available from the driver");
  g_encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
  fn = nullptr;
  YB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres));
  YB_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess,
             "cuTensorMapEncodeIm2col not available from the driver");
  g_encode_im2col = reinterpret_cast<EncodeIm2colFn>(fn);
  return YB_OK;
}

CUtensorMapSwizzle swizzle_for_row_bytes(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// wgmma N of an output tile: the next power of two >= 16 (weight rows past Cout_pad are zero-filled by the TMA unit, the
// store clips columns past Cout)
int mma_n(int n) {
  int c = 16;
  while (c < n) c <<= 1;
  return c;
}

}  // namespace

using ConvKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                              const ConvKernelParams);

// One kernel per (dtype, N tile, fused decode, chained tail N): the MMA width and the accumulator size are compile-time
// constants of every instance, so the accumulators stay in registers while the wgmma instructions are in flight.
// conv_configure admits exactly these shapes.
template <bool kBf16>
ConvKernelFn select_conv_kernel_t(const ConvKernelParams& kp) {
  if (kp.decode_on) return conv_wgmma_kernel<kBf16, 256, true, 0>;
  if (kp.ch.on) {
    if (kp.block_n == 64)
      return kp.ch.n2 == 32 ? conv_wgmma_kernel<kBf16, 64, false, 32>
                            : (kp.ch.n2 == 64 ? conv_wgmma_kernel<kBf16, 64, false, 64> : conv_wgmma_kernel<kBf16, 64, false, 128>);
    return kp.ch.n2 == 32 ? conv_wgmma_kernel<kBf16, 128, false, 32>
                          : (kp.ch.n2 == 64 ? conv_wgmma_kernel<kBf16, 128, false, 64> : conv_wgmma_kernel<kBf16, 128, false, 128>);
  }
  switch (kp.block_n) {
    case 16: return conv_wgmma_kernel<kBf16, 16, false, 0>;
    case 32: return conv_wgmma_kernel<kBf16, 32, false, 0>;
    case 64: return conv_wgmma_kernel<kBf16, 64, false, 0>;
    case 128: return conv_wgmma_kernel<kBf16, 128, false, 0>;
    default: return conv_wgmma_kernel<kBf16, 256, false, 0>;
  }
}
ConvKernelFn select_conv_kernel(const ConvKernelParams& kp) {
  return kp.ep.is_bf16 ? select_conv_kernel_t<true>(kp) : select_conv_kernel_t<false>(kp);
}

struct ConvOp {
  PatchConvOp* patch = nullptr;  // non-null: this conv runs on the halo-patch kernel
  CUtensorMap tmap_a, tmap_b, tmap_out, tmap_w2, tmap_out2;
  ConvKernelParams kp;
  ConvKernelFn fn = nullptr;
  dim3 grid;
  size_t smem_bytes;
};

// Pure host logic: validates the op and derives tiling, pipeline depth, shared-memory layout and launch shape
// (no driver calls: yb_conv_chain_supported runs this without a GPU).
static int conv_configure(const yb_op_desc& d, ConvKernelParams& kp, dim3& grid, size_t& smem_bytes) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "conv: dtype must be f16 or bf16");
  YB_REQUIRE((d.reserved & ~15) == 0, "conv: reserved bits 4 and up must be zero, got 0x%x", d.reserved);
  YB_REQUIRE(d.ksize >= 1 && d.ksize <= 7 && d.stride >= 1 && d.stride <= 2, "conv: ksize/stride");
  YB_REQUIRE(d.act >= YB_ACT_NONE && d.act <= YB_ACT_LEAKY01, "conv: unknown activation %d", d.act);
  YB_REQUIRE(d.Cin % 8 == 0 && d.in_cstride % 8 == 0 && d.in_cstride >= d.Cin,
             "conv: Cin/in_cstride must be multiples of 8 (16-byte TMA granularity), got %d/%d", d.Cin,
             d.in_cstride);
  YB_REQUIRE(d.Cout % 8 == 0 && d.out_cstride % 8 == 0 && d.out_cstride >= d.Cout,
             "conv: Cout/out_cstride must be multiples of 8, got %d/%d", d.Cout, d.out_cstride);
  YB_REQUIRE(d.Cin_pad % 16 == 0 && d.Cin_pad >= d.Cin, "conv: Cin_pad must be a multiple of 16");
  YB_REQUIRE(d.Cout_pad % 16 == 0 && d.Cout_pad >= d.Cout, "conv: Cout_pad must be a multiple of 16");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(d.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(d.weight) & 15) == 0,
             "conv: tensors must be 16-byte aligned");
  YB_REQUIRE(d.residual == nullptr ||
                 ((reinterpret_cast<uintptr_t>(d.residual) & 15) == 0 && d.res_cstride % 8 == 0),
             "conv: residual alignment");
  const int Ho = (d.H + 2 * d.pad - d.ksize) / d.stride + 1;
  const int Wo = (d.W + 2 * d.pad - d.ksize) / d.stride + 1;
  YB_REQUIRE(Ho == d.Ho && Wo == d.Wo, "conv: output extent mismatch (%d,%d) vs (%d,%d)", Ho, Wo, d.Ho,
             d.Wo);
  const long long M_ll = static_cast<long long>(d.N) * Ho * Wo;
  YB_REQUIRE(M_ll > 0 && M_ll < (1ll << 31), "conv: M out of range");

  YB_REQUIRE(!(d.reserved & 2) || patch_conv_eligible(d),
             "conv: banded stem weights (reserved bit 1) need the halo-patch kernel, which this %dx%d map does not qualify for",
             d.H, d.W);
  if (patch_conv_eligible(d)) return YB_OK;   // configured by patch_conv_configure
  kp = ConvKernelParams();
  kp.M = static_cast<int>(M_ll);
  kp.ep.Cout = d.Cout;
  const int m_tiles = (kp.M + kBlockM - 1) / kBlockM;
  const int sms = num_sms();
  // N tile: the whole Cout up to 256 columns (fewest A re-reads); halve it when that leaves fewer
  // than two tiles per SM so the persistent grid balances better.
  int n_tiles = (d.Cout + kMaxBlockN - 1) / kMaxBlockN;
  int block_n = mma_n((d.Cout + n_tiles - 1) / n_tiles);
  if (m_tiles * n_tiles < 2 * sms && block_n > 128 && d.chain == nullptr) block_n /= 2;
  n_tiles = (d.Cout + block_n - 1) / block_n;
  YB_REQUIRE(mma_n(block_n) == block_n && block_n <= kMaxBlockN, "conv: N tile %d is not a wgmma N", block_n);
  kp.block_n = block_n;
  kp.n_tiles = n_tiles;
  kp.num_tiles = m_tiles * n_tiles;
  kp.block_k = (d.Cin_pad % 64 == 0) ? 64 : ((d.Cin_pad % 32 == 0) ? 32 : 16);
  kp.ksize = d.ksize;
  kp.chunks = d.Cin_pad / kp.block_k;
  kp.num_k_iters = d.ksize * d.ksize * kp.chunks;
  kp.mode = (d.ksize == 1 && d.stride == 1 && d.pad == 0) ? 0 : 1;
  kp.HoWo = Ho * Wo;
  kp.Wo = Wo;
  kp.stride = d.stride;
  kp.pad = d.pad;
  kp.decode_on = 0;
  if (d.decode != nullptr) {
    const yb_head_decode& dd = *d.decode;
    const int width = dd.n_anchors * (dd.n_classes + 5);
    if (!(dd.n_anchors > 0 && dd.n_anchors <= 4 && width <= kMaxBlockN && width <= d.Cout_pad && d.ksize == 1 &&
          dd.keys && dd.boxes && dd.img_count && dd.img_maxc)) {
      set_error("conv: fused decode needs a 1x1 head with n_anchors*(n_classes+5) <= %d and a candidate arena", kMaxBlockN);
      return YB_ERR_INVALID;
    }
    // all anchors of a pixel must sit in one accumulator row: one N tile covering the whole head
    n_tiles = 1;
    block_n = mma_n(d.Cout);
    YB_REQUIRE(block_n == 256, "conv: the fused decode is built for heads of 129-256 columns, got %d", d.Cout);
    kp.block_n = block_n;
    kp.n_tiles = 1;
    kp.num_tiles = m_tiles;
    kp.decode_on = 1;
    kp.dec = dd;
    kp.dec_H = Ho;
    kp.dec_W = Wo;
  }
  kp.store_cols = (block_n % 64 == 0) ? 64 : ((block_n % 32 == 0) ? 32 : 16);
  kp.bias_len = d.Cout_pad;
  kp.kk_last = (d.Cin - (kp.chunks - 1) * kp.block_k + 15) / 16;
  if (kp.kk_last < 1) kp.kk_last = 1;
  if (kp.kk_last > (kp.block_k >> 4)) kp.kk_last = kp.block_k >> 4;
  kp.a_stage_bytes = kBlockM * kp.block_k * 2;
  kp.b_stage_bytes = (static_cast<uint32_t>(kp.block_n * kp.block_k * 2) + 1023u) & ~1023u;
  kp.ch.on = 0;
  size_t chain_bytes = 0;
  if (d.chain != nullptr) {
    YB_REQUIRE(kp.store_cols == 64, "conv: a chained tail needs 64-column output boxes (Cout %% 64 == 0), got Cout=%d", d.Cout);
    const char* why = chain_setup(d, kp.block_n, kp.n_tiles, kp.store_cols, /*allow_extra=*/false, &kp.ch);
    YB_REQUIRE(why == nullptr, "conv: chained tail not supported here: %s", why);
    const int s2 = chain_store2_cols(kp.ch.n2);
    YB_REQUIRE(s2 == 64 || s2 == 32, "conv: the tail's Cout_pad must be a multiple of 32, got %d", kp.ch.n2);
    YB_REQUIRE((kp.block_n == 64 || kp.block_n == 128) && kp.ch.n2 <= 128,
               "conv: chained tails are built for N tiles of 64 / 128 and tails of at most 128 columns (block_n=%d, n2=%d)",
               kp.block_n, kp.ch.n2);
    chain_bytes = static_cast<size_t>(kp.ch.w2_chunks) * kp.ch.w2_sub_bytes;
  }
  // Weights stay resident in shared memory when the layer has a single N tile and they are small:
  // the persistent CTA then streams only activations (halves the L2->SM traffic of the shallow layers).
  const size_t fixed = static_cast<size_t>(kStageBufs) * kStageBufBytes + 1024 + chain_bytes;
  const size_t b_total = static_cast<size_t>(kp.num_k_iters) * kp.b_stage_bytes;
  kp.b_resident = (n_tiles == 1 && b_total <= 80 * 1024) ? 1 : 0;
  kp.b_res_bytes = kp.b_resident ? static_cast<uint32_t>(b_total) : 0u;
  // k-iterations per pipeline stage: aim at ~32 KB per stage so that one mbarrier round trip moves
  // enough bytes (a 16-channel tap is only 4 KB), in near-equal groups.
  const uint32_t per_iter = kp.a_stage_bytes + (kp.b_resident ? 0u : kp.b_stage_bytes);
  YB_REQUIRE(kSmemBudget > fixed + kp.b_res_bytes + 2 * per_iter, "conv: shared memory budget exceeded (block_n=%d)", kp.block_n);
  const size_t avail = kSmemBudget - fixed - kp.b_res_bytes;
  const size_t target = avail / 3 < 32 * 1024 ? avail / 3 : 32 * 1024;   // keep at least three stages in flight
  int kpg_max = static_cast<int>(target / per_iter);
  if (kpg_max < 1) kpg_max = 1;
  if (kpg_max > kp.num_k_iters) kpg_max = kp.num_k_iters;
  const int groups = (kp.num_k_iters + kpg_max - 1) / kpg_max;
  kp.kpg = (kp.num_k_iters + groups - 1) / groups;
  const uint32_t stage_bytes = kp.kpg * per_iter;
  int stages = static_cast<int>(avail / stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  kp.stages = stages;
  kp.ep.is_bf16 = d.dtype == YB_BF16;
  kp.ep.act = d.act;
  kp.bias = d.bias;
  kp.ep.residual = d.residual;
  kp.ep.res_cstride = d.res_cstride;
  grid = dim3(kp.num_tiles < sms ? kp.num_tiles : sms, 1, 1);
  const size_t smem = static_cast<size_t>(stages) * stage_bytes + kp.b_res_bytes + fixed;
  YB_REQUIRE(smem <= kSmemBudget, "conv: %zu bytes of shared memory needed, %zu available", smem, kSmemBudget);
  smem_bytes = smem;
  return YB_OK;
}

int conv_configure_check(const yb_op_desc& d, int* info) {
  ConvKernelParams kp;
  dim3 grid;
  size_t smem = 0;
  const int rc = conv_configure(d, kp, grid, smem);
  if (rc == YB_OK && info && !patch_conv_eligible(d)) {   // yb_conv_config: see include/yolort_b200.h
    info[0] = 0;
    info[1] = kp.block_n;
    info[2] = kp.n_tiles;
    info[3] = kp.b_resident;
    info[4] = 1;
    info[5] = kp.stages;
    info[6] = kp.kpg;
    info[7] = kp.store_cols;
    info[8] = kConsumers;         // (im2col / 1x1 kernel: consumer warpgroups; they share two staging buffers)
    info[9] = static_cast<int>(smem);
    info[10] = static_cast<int>(grid.x);
    info[11] = kp.ch.on;
  }
  return rc;
}

int conv_op_create(const yb_op_desc& d, ConvOp** out) {
  int rc = load_driver_entry_points();
  if (rc != YB_OK) return rc;
  ConvOp* op = new ConvOp();
  rc = conv_configure(d, op->kp, op->grid, op->smem_bytes);
  if (rc != YB_OK) {
    delete op;
    return rc;
  }
  if (patch_conv_eligible(d)) {
    rc = patch_conv_create(d, g_encode_tiled, &op->patch);
    if (rc != YB_OK) {
      delete op;
      return rc;
    }
    *out = op;
    return YB_OK;
  }
  ConvKernelParams& kp = op->kp;
  const int Ho = d.Ho, Wo = d.Wo;
  (void)Ho; (void)Wo;

  const CUtensorMapDataType dt =
      kp.ep.is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const CUtensorMapSwizzle sw = swizzle_for_row_bytes(kp.block_k * 2);
  CUresult cr;
  if (kp.mode == 0) {
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(kp.M)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.in_cstride) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(kp.block_k), kBlockM};
    cuuint32_t estr[2] = {1, 1};
    cr = g_encode_tiled(&op->tmap_a, dt, 2, const_cast<void*>(d.in), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(d.W),
                          static_cast<cuuint64_t>(d.H), static_cast<cuuint64_t>(d.N)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(d.in_cstride) * 2,
                             static_cast<cuuint64_t>(d.in_cstride) * 2 * d.W,
                             static_cast<cuuint64_t>(d.in_cstride) * 2 * d.W * d.H};
    int lower[2] = {-d.pad, -d.pad};
    int upper[2] = {d.pad - (d.ksize - 1), d.pad - (d.ksize - 1)};
    cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(d.stride), static_cast<cuuint32_t>(d.stride), 1};
    cr = g_encode_im2col(&op->tmap_a, dt, 4, const_cast<void*>(d.in), dims, strides, lower, upper,
                         static_cast<cuuint32_t>(kp.block_k), kBlockM, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    // Driver workaround also applied by CUTLASS (copy_traits_sm90_im2col.hpp): for tensors smaller
    // than 128 KiB, drivers <= 13.1 set a descriptor bit that makes im2col loads fault.
    int drv = 0;
    cudaDriverGetVersion(&drv);
    const size_t span = static_cast<size_t>(d.in_cstride) * 2 * d.W * d.H * d.N;
    if (cr == CUDA_SUCCESS && drv <= 13010 && span < 131072) {
      reinterpret_cast<uint64_t*>(&op->tmap_a)[1] &= ~(1ull << 21);
    }
  }
  if (cr != CUDA_SUCCESS) {
    set_error("conv: cuTensorMapEncode (A, mode %d) failed with CUresult %d (Cin=%d cs=%d H=%d W=%d N=%d k=%d s=%d bk=%d)",
              kp.mode, static_cast<int>(cr), d.Cin, d.in_cstride, d.H, d.W, d.N, d.ksize, d.stride,
              kp.block_k);
    delete op;
    return YB_ERR_CUDA;
  }
  {
    const int ktot = d.ksize * d.ksize * d.Cin_pad;
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(ktot), static_cast<cuuint64_t>(d.Cout_pad)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ktot) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(kp.block_k), static_cast<cuuint32_t>(kp.block_n)};
    cuuint32_t estr[2] = {1, 1};
    cr = g_encode_tiled(&op->tmap_b, dt, 2, const_cast<void*>(d.weight), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("conv: cuTensorMapEncodeTiled (weights) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  {
    // destination view [M rows, Cout channels], row pitch = out_cstride; boxes of 128 rows x store_cols
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.Cout), static_cast<cuuint64_t>(kp.M)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.out_cstride) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(kp.store_cols), kBlockM};
    cuuint32_t estr[2] = {1, 1};
    cr = g_encode_tiled(&op->tmap_out, dt, 2, d.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_for_row_bytes(kp.store_cols * 2), CU_TENSOR_MAP_L2_PROMOTION_NONE,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("conv: cuTensorMapEncodeTiled (output) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  op->tmap_w2 = op->tmap_b;      // placeholders when nothing is chained (never dereferenced)
  op->tmap_out2 = op->tmap_out;
  if (kp.ch.on) {
    const yb_conv_chain& c = *d.chain;
    const int kc = kp.ch.w2_row_bytes / 2;
    cuuint64_t wdims[2] = {static_cast<cuuint64_t>(c.K_pad), static_cast<cuuint64_t>(c.Cout_pad)};
    cuuint64_t wstrides[1] = {static_cast<cuuint64_t>(c.K_pad) * 2};
    cuuint32_t wbox[2] = {static_cast<cuuint32_t>(kc), static_cast<cuuint32_t>(kp.ch.n2)};
    cuuint32_t estr[2] = {1, 1};
    cr = g_encode_tiled(&op->tmap_w2, dt, 2, const_cast<void*>(c.weight), wdims, wstrides, wbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_for_row_bytes(kc * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr == CUDA_SUCCESS) {
      const int s2 = chain_store2_cols(kp.ch.n2);
      cuuint64_t odims[2] = {static_cast<cuuint64_t>(c.Cout), static_cast<cuuint64_t>(kp.M)};
      cuuint64_t ostrides[1] = {static_cast<cuuint64_t>(c.out_cstride) * 2};
      cuuint32_t obox[2] = {static_cast<cuuint32_t>(s2), kBlockM};
      cr = g_encode_tiled(&op->tmap_out2, dt, 2, c.out, odims, ostrides, obox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          swizzle_for_row_bytes(s2 * 2), CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (cr != CUDA_SUCCESS) {
      set_error("conv: cuTensorMapEncodeTiled (chained tail) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  op->fn = select_conv_kernel(kp);
  cudaError_t e = cudaFuncSetAttribute(op->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBudget));
  if (e != cudaSuccess) {
    set_error("conv: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    delete op;
    return YB_ERR_CUDA;
  }
  *out = op;
  return YB_OK;
}

int conv_op_launch(const ConvOp* op, cudaStream_t stream) {
  if (op->patch) return patch_conv_launch(op->patch, stream);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = op->grid;
  cfg.blockDim = dim3(kThreads, 1, 1);
  cfg.dynamicSmemBytes = op->smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  YB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, op->fn, op->tmap_a, op->tmap_b, op->tmap_out, op->tmap_w2, op->tmap_out2, op->kp));
  return YB_OK;
}

void conv_op_destroy(ConvOp* op) {
  if (op && op->patch) patch_conv_destroy(op->patch);
  delete op;
}

}  // namespace yb
