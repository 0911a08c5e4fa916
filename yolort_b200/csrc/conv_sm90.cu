// Conv2d(+folded BN)+SiLU(+residual) as an implicit GEMM on the Hopper tensor cores (wgmma).
//
//   D[m, co] = sum_{r,s,ci} X[n, ho*stride - pad + r, wo*stride - pad + s, ci] * W[co, r, s, ci]
//   m = (n*Ho + ho)*Wo + wo      (NHWC activations, K-major weights)
//
// Replaces the arithmetic of yolort/v5/models/common.py:42-73 (Conv = conv2d -> BN(eps 1e-3) -> SiLU),
// :94-116 (Bottleneck residual) and the 1x1 head convs of yolort/models/box_head.py:35-37,68-82.
//
// Persistent kernel, one CTA per SM (two for the narrow shallow layers, see conv_configure), static round-robin over
// 128 x block_n output tiles, 384 threads:
//   warpgroup 0 (producer, 40 registers): warp 0 issues the TMA loads.  A tiles come from a 4-D im2col tensor map (the
//                TMA engine walks 128 output pixels, applies padding/stride and zero-fills the halo) or, for 1x1/s1
//                convs, from a 2-D tiled map; B tiles (weights) from a 2-D tiled map.  Both land in shared memory in the
//                32/64/128-byte swizzled K-major layout wgmma reads.  The producer runs ahead across tile boundaries.
//   warpgroups 1-2 (consumers, 232 registers): each multiplies 64 rows of the tile (wgmma m64nNk16, N = block_n, fp32
//                accumulators in registers), then runs the epilogue on its fragment: +bias -> activation -> (+residual)
//                -> fp16/bf16 -> swizzled shared-memory staging -> TMA store into the NHWC destination view (a channel
//                window of a concat buffer is just a strided tensor map; ragged M is clipped by the TMA unit).
// Instances with ONE consumer warpgroup (256 threads, 64-row tiles, two CTAs per SM at the consumers' 232 registers) run
// the same protocol with half the participants: the two co-resident CTAs take the place of the two consumer warpgroups,
// and one CTA's epilogue overlaps the other's MMAs.  The large chained 1x1 launches at N = 128, whose resident weights
// leave room for one CTA per SM only, run on a lean 640-thread instance: two teams of two consumer warpgroups take the
// CTA's tiles alternately, so one team's epilogue and chained tail overlap the other team's MMAs
// (conv_wgmma_team_kernel).  The deep launches that stream their weights run on a 640-thread instance too: a task is two
// 128-row tiles that share every weight slab, so each slab crosses from L2 once per two tiles (conv_wgmma_quad_kernel).
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

constexpr int kMaxStages = 12;
// consumer warpgroups per CTA (64 accumulator rows each): 2, or 1 in the 64-row-tile instances
__host__ __device__ constexpr int tile_rows(int groups) { return 64 * groups; }
__host__ __device__ constexpr int cta_threads(int groups) { return 128 * (1 + groups); }
// staging box: the tile's rows x (up to) 64 columns x 2 B
__host__ __device__ constexpr int stage_buf_bytes(int groups) { return tile_rows(groups) * 128; }
constexpr int kStageBufs = 2;              // staging boxes, shared by the consumer warpgroups
constexpr int kMaxBlockN = 256;
constexpr size_t kSmemBudget = 216 * 1024;  // dynamic shared memory per CTA (227 KB limit minus static)
constexpr size_t kStaticSmem = (2 * kMaxStages + 2) * 8 + 2 * kMaxBlockN * 4;   // barriers + bias vectors (ptxas -v)
constexpr uint32_t kConsumerBar = 1;        // named barrier of the consumer threads

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
  // Split tail: the tasks from full_tiles on are the last round's r = num_tiles - full_tiles tiles, each cut into `split`
  // halves (kernel: 64-row or 64-column; split = 1: num_tasks = num_tiles, every task a whole tile)
  int full_tiles, split, num_tasks;
  int ctas;        // CTAs per SM the launch is planned for (1 or 2): selects the kernel instance
  int groups;      // consumer warpgroups per CTA (2, 1 with two CTAs per SM, or 4): selects the kernel instance
  int pair;        // M tiles per task: 1, or 2 when two tiles share each streamed weight slab (conv_quad_plan)
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

template <int kGroups>
__device__ __forceinline__ void consumer_sync() { named_bar_sync(kConsumerBar, 128 * kGroups); }

// Task t of the grid's walk: its tile's M tile and N tile, and which of the tile's `split` halves it computes
// (piece 0 of 1 for a whole tile).  The tail sub-tasks are ordered so that task full_tiles + u, which CTA u runs, lies
// in N tile u % n_tiles: a CTA keeps the N tile (and resident weights) of its full rounds, as the grid and full_tiles are
// multiples of n_tiles (conv_plan).  Instances without tail halves (kSplits false) walk whole tiles only.
struct ConvTask {
  int m_tile, n_tile, piece, split;
};
template <bool kSplits>
__device__ __forceinline__ ConvTask conv_task(const ConvKernelParams& p, int t) {
  ConvTask k;
  int tile = t;
  k.piece = 0;
  k.split = 1;
  if (kSplits && t >= p.full_tiles) {
    const int u = t - p.full_tiles;
    const int q = u / p.n_tiles;
    tile = p.full_tiles + (q / p.split) * p.n_tiles + (u - q * p.n_tiles);
    k.piece = q % p.split;
    k.split = p.split;
  }
  k.m_tile = tile / p.n_tiles;
  k.n_tile = tile - k.m_tile * p.n_tiles;
  return k;
}

// One pipeline stage's MMAs at the wgmma N kW (the tile's kN, or a tail half's kN / 2): `cnt` k-iterations
// of A and B sub-tiles; returns the channel chunk the next stage starts at.
template <bool kBf16, int kW>
__device__ __forceinline__ int stage_mmas(float* acc, const ConvKernelParams& p, uint32_t a_lo0, uint32_t a_step16,
                                          uint32_t b_lo0, uint32_t b_step16, uint64_t ab_hi, int cnt, int ch, int kk,
                                          bool first) {
  for (int j = 0; j < cnt; ++j) {
    const int kc = ch == p.chunks - 1 ? p.kk_last : kk;
    for (int k = 0; k < kc; ++k)
      wgmma_mma<kBf16, kW>(acc, desc_lohi(a_lo0 + j * a_step16 + 2 * k, ab_hi), desc_lohi(b_lo0 + j * b_step16 + 2 * k, ab_hi),
                           !first || (j | k) != 0);
    if (++ch == p.chunks) ch = 0;
  }
  return ch;
}

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
// pointwise tail is chained onto every tile (conv_chain.cuh).  kCtas: CTAs resident per SM (1 or 2, see
// regs_producer); with two, one CTA's epilogue and barrier waits overlap the other CTA's MMAs and loads.  kGroups:
// consumer warpgroups per CTA (2: 128-row tiles; 1: 64-row tiles, two CTAs per SM with 232 consumer registers).
template <bool kBf16, int kN, bool kDecode, int kN2, int kCtas, int kGroups = 2>
__global__ void __launch_bounds__(cta_threads(kGroups), kCtas)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_w2,
                  const __grid_constant__ CUtensorMap tmap_out2, const __grid_constant__ CUtensorMap tmap_a64,
                  const __grid_constant__ CUtensorMap tmap_out64, const ConvKernelParams p) {
  static_assert(kGroups == 2 || (kGroups == 1 && kCtas == 2 && !kDecode), "one consumer warpgroup: two CTAs, no decode");
  constexpr bool kChain = kN2 != 0;
  constexpr int kAcc = (kN > kN2 ? kN : kN2) / 2;   // accumulator registers per thread
  constexpr int kBlockM = tile_rows(kGroups);
  constexpr int kStageBufBytes = stage_buf_bytes(kGroups);
  // Tail halves in the 128-column instances only (the N = 256 instances spill their 128 accumulators with any of this
  // code).  With two consumer warpgroups a half is 64 rows of the tile: both warpgroups multiply the same 64 A rows,
  // each with its 64 columns of the tile, so the sub-task loads half the tile's A.  With one warpgroup (64-row tiles) a
  // half is 64 columns of the tile.
  constexpr bool kSplits = !kDecode && !kChain && kN == 128;
  constexpr bool kRowHalves = kSplits && kGroups == 2;
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
      mbar_init(&empty_bar[s], kGroups);   // one arrival per consumer warpgroup
    }
    mbar_init(&b_full, 1);
    mbar_init(&w2_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // Programmatic dependent launch: everything above overlapped the tail of the previous kernel in the stream.
  // Resident weights do not depend on the previous kernel: their loads are issued BEFORE the grid-dependency wait
  // and stream in while the previous kernel drains.
  if (threadIdx.x == 0 && p.b_resident) {   // the CTA's one N tile (conv_plan: the grid is a multiple of n_tiles)
    const uint32_t b_bytes = p.block_n * p.block_k * 2;
    const int n0 = (blockIdx.x % p.n_tiles) * p.block_n;
    mbar_expect_tx(&b_full, p.num_k_iters * b_bytes);
    for (int it = 0; it < p.num_k_iters; ++it)
      tma_load_2d(&tmap_b, &b_full, b_res + it * p.b_stage_bytes, it * p.block_k, n0);
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
    regs_producer<kCtas, kGroups>();
    if (warp != 0) return;
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    const uint32_t a_bytes = kBlockM * p.block_k * 2, b_bytes = p.block_n * p.block_k * 2;
    int kit = 0;
    for (int t = blockIdx.x; t < p.num_tasks; t += gridDim.x) {
      const ConvTask task = conv_task<kSplits>(p, t);   // a tail half loads the whole tile's B
      const bool rows64 = kRowHalves && task.split != 1;   // a row half: 64 A rows through the 64-row map
      const int n0 = task.n_tile * p.block_n;
      const int m0 = task.m_tile * kBlockM + (rows64 ? task.piece * 64 : 0);
      const CUtensorMap* map_a = rows64 ? &tmap_a64 : &tmap_a;
      const uint32_t a_task_bytes = rows64 ? a_bytes / 2 : a_bytes;
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
          mbar_expect_tx(&full_bar[s], cnt * (a_task_bytes + (p.b_resident ? 0u : b_bytes)));
          for (int j = 0; j < cnt; ++j) {
            const int it = it0 + j;
            const int tap = it / p.chunks;
            const int chunk = it - tap * p.chunks;
            if (p.mode == 0) {
              tma_load_2d(map_a, &full_bar[s], a_dst + j * p.a_stage_bytes, chunk * p.block_k, m0);
            } else {
              const int r = tap / p.ksize;
              const int sx = tap - r * p.ksize;
              tma_load_im2col_4d(map_a, &full_bar[s], a_dst + j * p.a_stage_bytes, chunk * p.block_k, cw, ch, cn,
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
  regs_consumer<kCtas, kGroups>();
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
    for (int i = ctid; i < p.ch.n2; i += 128 * kGroups) s_bias2[i] = (i < p.ch.bias2_len) ? __ldg(p.ch.bias2 + i) : 0.f;
  }
  // Every tile of this CTA has the same N tile when the grid is a multiple of the N-tile count (always with one N
  // tile): the bias is then loaded ONCE instead of per tile.
  const bool fixed_n = (gridDim.x % p.n_tiles) == 0;
  if (fixed_n) {
    const int n0f = (blockIdx.x % p.n_tiles) * p.block_n;
    for (int i = ctid; i < p.block_n; i += 128 * kGroups) s_bias[i] = (n0f + i < p.bias_len) ? __ldg(p.bias + n0f + i) : 0.f;
  }
  consumer_sync<kGroups>();
  if (p.b_resident) mbar_wait(&b_full, 0);
  if constexpr (kChain) mbar_wait(&w2_full, 0);

  int kit = 0, store_idx = 0;
  for (int t = blockIdx.x; t < p.num_tasks; t += gridDim.x) {
    const ConvTask task = conv_task<kSplits>(p, t);
    const bool half = kSplits && task.split != 1;
    const bool rows64 = kRowHalves && half;
    const int width = half ? bn / 2 : bn;   // columns this warpgroup computes and stores
    // this warpgroup's first column in the tile: a column half's, or (row halves) the warpgroup's half of the columns
    const int col0 = half ? (rows64 ? g : task.piece) * width : 0;
    const int n0 = task.n_tile * p.block_n + col0;
    const int m0 = task.m_tile * kBlockM + (rows64 ? task.piece * 64 : 0);
    const bool load_bias = !fixed_n || (half && !rows64);   // s_bias holds the task's columns from s_bias[0]
    if (load_bias) {
      consumer_sync<kGroups>();   // the previous tile's epilogue has finished with the bias (and the staging boxes)
      const int nb = rows64 ? n0 - col0 : n0, wb = rows64 ? bn : width;
      for (int i = ctid; i < wb; i += 128 * kGroups) s_bias[i] = (nb + i < p.bias_len) ? __ldg(p.bias + nb + i) : 0.f;
    }
    const float* bias_cols = s_bias + (rows64 ? col0 : 0);
    // the task's rows of the tile's B sub-tiles (multiples of 64 rows keep the 8-row swizzle phase); a row half's two
    // warpgroups read the same 64 A rows
    const uint32_t b_piece16 = (col0 * row_bytes) >> 4;
    const uint32_t a_group16 = rows64 ? 0u : g * a_half16;

    // ---- main loop: stage s is released once the MMAs that read it have completed (one stage in flight) ----
    int chunk = 0, prev_s = -1;
    for (int it0 = 0; it0 < p.num_k_iters; it0 += p.kpg, ++kit) {
      const int cnt = min(p.kpg, p.num_k_iters - it0);
      const int s = kit % p.stages;
      mbar_wait(&full_bar[s], (kit / p.stages) & 1);
      const uint32_t a_lo0 = smem_lo16(tiles + s * stage_bytes) + a_group16;
      const uint32_t b_lo0 =
          (p.b_resident ? b_res_lo0 + it0 * b_step16 : smem_lo16(tiles + s * stage_bytes) + p.kpg * a_step16) + b_piece16;
      wgmma_fence();
      int ch;
      if (!kSplits || width == bn)
        ch = stage_mmas<kBf16, kN>(acc, p, a_lo0, a_step16, b_lo0, b_step16, ab_hi, cnt, chunk, kk, it0 == 0);
      else
        ch = stage_mmas<kBf16, kSplits ? kN / 2 : kN>(acc, p, a_lo0, a_step16, b_lo0, b_step16, ab_hi, cnt, chunk, kk, it0 == 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_s >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
      chunk = ch;
    }
    wgmma_wait<0>();
    fence_acc<kN / 2>(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_s]);
    if (load_bias) consumer_sync<kGroups>();   // bias visible

    // fr.loc is the row in the staging box; a row half's warpgroups both hold rows m0 .. m0 + 63
    fr.row[0] = static_cast<long long>(m0) + fr.loc[0] - (rows64 ? g * 64 : 0);
    fr.row[1] = static_cast<long long>(m0) + fr.loc[1] - (rows64 ? g * 64 : 0);
    fr.ok[0] = fr.row[0] < p.M;
    fr.ok[1] = fr.row[1] < p.M;
    if constexpr (kDecode) {
      decode_fragment<kN>(p.dec, acc, s_bias, fr, p.dec_H, p.dec_W, reinterpret_cast<float*>(staging), 2 + g, lane);
    } else {
    if constexpr (kChain) {
      // chain tiles index the staging buffers by box (box b of the tile stays in buffer b until the tail GEMM has read
      // it), so the previous tile's stores must have drained both buffers before this tile writes them
      if (issuer) tma_store_wait_read<0>();
      consumer_sync<kGroups>();
    }
    for (int c0 = 0; c0 < width; c0 += store_cols, ++store_idx) {
      // Two staging buffers, one barrier per box: before the barrier below the issuer waits until the PREVIOUS
      // store has finished reading its buffer, which is the one the next box will overwrite.
      uint8_t* buf = staging + (kChain ? (c0 / store_cols) : (store_idx & 1)) * kStageBufBytes;
      epilogue_box<kBf16, kN>(p.ep, acc, c0, store_cols, bias_cols, fr, n0, buf, lane);
      fence_proxy_async_smem();
      if constexpr (!kChain) {
        if (issuer) tma_store_wait_read<0>();
      }
      consumer_sync<kGroups>();
      if (issuer) {
        if (rows64) {   // each warpgroup's 64 x 64 box: rows 0-63 / 64-127 of the staging buffer
          const int nt = task.n_tile * p.block_n;
          if (m0 < p.M) {
            if (nt + c0 < p.ep.Cout) tma_store_2d(&tmap_out64, buf, nt + c0, m0);
            if (nt + width + c0 < p.ep.Cout) tma_store_2d(&tmap_out64, buf + 64 * store_cols * 2, nt + width + c0, m0);
          }
        } else if ((!kChain || p.ch.store_first) && n0 + c0 < p.ep.Cout) {
          tma_store_2d(&tmap_out, buf, n0 + c0, m0);
        }
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
      consumer_sync<kGroups>();
      const int s2 = chain_store2_cols(p.ch.n2);
      for (int c0 = 0; c0 < p.ch.n2; c0 += s2) {
        uint8_t* buf = staging + ((c0 / s2) & 1) * kStageBufBytes;
        epilogue_box<kBf16, kChain ? kN2 : 16>(p.ch.ep2, acc, c0, s2, s_bias2, fr, 0, buf, lane);
        fence_proxy_async_smem();
        if (issuer) tma_store_wait_read<0>();   // box k + 1 overwrites the buffer of box k - 1
        consumer_sync<kGroups>();
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

// ===================== two consumer teams: chained 1x1 tiles over one resident weight copy =====================
// The large one-CTA chained 1x1 launches (C3's cv1 || cv2 -> m.0.cv1 at N = 128 with a 64-column tail): their resident
// weights leave room for one CTA per SM only, and on that CTA's two consumer warpgroups nothing issued MMAs while a tile
// ran its epilogue boxes, its store waits, the tail GEMM and the tail epilogue.  This lean instance has one producer
// warpgroup and four consumer warpgroups (640 threads); warpgroups 2t + 1 and 2t + 2 form team t, which owns a whole
// 128-row tile and runs on it exactly the chain path of conv_wgmma_kernel.  Team t takes positions t, t + 2, ... of the
// CTA's tile list, so one team's epilogue and tail overlap the other team's MMAs.  Shared: the resident weights, the
// resident tail weights, both bias vectors and the producer warp; per team: a named barrier (2 + t; the 512 consumer
// threads use kConsumerBar), two 16 KB staging boxes, a TMA-store issuer whose bulk async-groups are its own, and an
// A ring of one-k-iteration stages.  The producer fills ring k & 1 with the CTA's k-th tile, so a team's parity wait
// on a slot always follows the fill it waited on last.  Every output element gets the k16 MMA sequence and the
// epilogue of conv_wgmma_kernel, so the outputs are the same bits.  Only what these launches need is compiled: mode 0
// (2-D tiled A), whole 64-channel K chunks, one N tile of resident weights, a chained tail of kN2 columns over one or
// two 64-channel staged boxes, no fused decode and no split tail.
constexpr int kTeamThreads = 640;
constexpr int kTeamMaxStages = 6;        // A stages per team
constexpr int kTeamMinTilesPerSm = 8;    // conv_team_plan
constexpr uint32_t kTeamBar0 = 2;        // team t syncs on named barrier 2 + t
constexpr size_t kTeamStaticSmem = (4 * kTeamMaxStages + 2) * 8 + 2 * 128 * 4;   // barriers + bias vectors
constexpr size_t kTeamSmemBudget = 227 * 1024 - kTeamStaticSmem;

template <bool kBf16, int kN, int kN2>
__global__ void __launch_bounds__(kTeamThreads, 1)
conv_wgmma_team_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_w2,
                       const __grid_constant__ CUtensorMap tmap_out2, const __grid_constant__ CUtensorMap tmap_a64,
                       const __grid_constant__ CUtensorMap tmap_out64, const ConvKernelParams p) {
  static_assert(kN == 128 && kN2 == 64, "team instances: N = 128 with a 64-column tail");
  constexpr int kStageBufBytes = stage_buf_bytes(2);
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[2][kTeamMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[2][kTeamMaxStages];
  __shared__ __align__(8) uint64_t b_full;
  __shared__ __align__(8) uint64_t w2_full;
  __shared__ __align__(16) float s_bias[kN];
  __shared__ __align__(16) float s_bias2[kN2];

  uint8_t* tiles = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const uint32_t ring_bytes = static_cast<uint32_t>(p.stages) * p.a_stage_bytes;   // [2 teams][stages][A sub-tile]
  uint8_t* b_res = tiles + 2 * ring_bytes;                  // resident weights
  uint8_t* staging = b_res + p.b_res_bytes;                 // [2 teams][kStageBufs][kStageBufBytes]
  uint8_t* w2_res = staging + 2 * kStageBufs * kStageBufBytes;   // resident tail weights

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int r = 0; r < 2; ++r) {
      for (int s = 0; s < p.stages; ++s) {
        mbar_init(&full_bar[r][s], 1);
        mbar_init(&empty_bar[r][s], 2);   // the two warpgroups of the team
      }
    }
    mbar_init(&b_full, 1);
    mbar_init(&w2_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  // the weights do not depend on the previous kernel: loaded before the grid-dependency wait, as conv_wgmma_kernel
  if (threadIdx.x == 0) {
    const uint32_t b_bytes = p.block_n * p.block_k * 2;
    mbar_expect_tx(&b_full, p.num_k_iters * b_bytes);
    for (int it = 0; it < p.num_k_iters; ++it) tma_load_2d(&tmap_b, &b_full, b_res + it * p.b_stage_bytes, it * p.block_k, 0);
    tma_prefetch_desc(&tmap_w2);
    tma_prefetch_desc(&tmap_out2);
    mbar_expect_tx(&w2_full, p.ch.w2_chunks * p.ch.n2 * p.ch.w2_row_bytes);
    for (int j = 0; j < p.ch.w2_chunks; ++j)
      tma_load_2d(&tmap_w2, &w2_full, w2_res + j * p.ch.w2_sub_bytes, j * (p.ch.w2_row_bytes >> 1), 0);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // 128 x 24 + 512 x 112 <= 640 x 96: the producers lower their budget and return before the consumers raise theirs
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (warp != 0) return;
    // ===================== A producer: the CTA's tiles in order, tile k into ring k & 1 =====================
    const uint32_t a_bytes = p.a_stage_bytes;
    int kit0 = 0, kit1 = 0;   // fills of each ring so far
    for (int t = blockIdx.x, k = 0; t < p.num_tiles; t += gridDim.x, ++k) {
      const int r = k & 1;
      const int m0 = t * 128;
      int kit = r ? kit1 : kit0;
      for (int it = 0; it < p.num_k_iters; ++it, ++kit) {
        const int s = kit % p.stages;
        mbar_wait(&empty_bar[r][s], ((kit / p.stages) & 1) ^ 1);
        if (YB_ELECT()) {
          mbar_expect_tx(&full_bar[r][s], a_bytes);
          tma_load_2d(&tmap_a, &full_bar[r][s], tiles + r * ring_bytes + s * a_bytes, it * p.block_k, m0);
        }
      }
      (r ? kit1 : kit0) = kit;
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 112;\n" ::: "memory");

  // ===================== consumers: team `team`, warpgroup `half` of it multiplies rows 64 half .. +63 =====================
  const int cw = (warp >> 2) - 1;
  const int team = cw >> 1, half = cw & 1;
  const int wq = warp & 3;
  const int ctid = threadIdx.x - 128;
  const bool issuer = (ctid & 255) == 0;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint32_t team_bar = kTeamBar0 + team;
  FragRows fr;
  fr.loc[0] = half * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  uint8_t* team_staging = staging + static_cast<size_t>(team) * kStageBufs * kStageBufBytes;
  uint8_t* ring = tiles + team * ring_bytes;
  float acc[kN / 2];

  for (int i = ctid; i < kN; i += 512) s_bias[i] = (i < p.bias_len) ? __ldg(p.bias + i) : 0.f;
  for (int i = ctid; i < kN2; i += 512) s_bias2[i] = (i < p.ch.bias2_len) ? __ldg(p.ch.bias2 + i) : 0.f;
  named_bar_sync(kConsumerBar, 512);
  mbar_wait(&b_full, 0);
  mbar_wait(&w2_full, 0);

  int kit = 0;
  for (int t = blockIdx.x + team * gridDim.x; t < p.num_tiles; t += 2 * gridDim.x) {
    const int m0 = t * 128;
    {
      // descriptor constants, derived per tile rather than held through the epilogue (registers are short)
      const uint32_t ab_hi = desc_hi(128, 8 * 128);                  // 64-channel rows of 128 bytes
      const uint32_t a_wg16 = (64 * 128 * half) >> 4;                // this warpgroup's 64 rows of an A sub-tile
      const uint32_t b_lo0 = smem_lo16(b_res);
      const uint32_t b_step16 = p.b_stage_bytes >> 4;
      // The first MMA overwrites the accumulators; zeroing them first tells ptxas that the previous tile's values are
      // dead, which it cannot see through the run-time accumulate flag (they would otherwise stay live across the tail
      // GEMM and spill).
#pragma unroll
      for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
      // ---- main loop: stage s is released once the MMAs that read it have completed (one stage in flight) ----
      int prev_s = -1;
      for (int it = 0; it < p.num_k_iters; ++it, ++kit) {
        const int s = kit % p.stages;
        mbar_wait(&full_bar[team][s], (kit / p.stages) & 1);
        const uint32_t a_lo = smem_lo16(ring + s * p.a_stage_bytes) + a_wg16;
        const uint32_t b_lo = b_lo0 + it * b_step16;
        wgmma_fence();
        // whole 64-channel chunks (conv_team_plan): four K steps, a fixed count (ptxas serialises the wgmmas of a
        // run-time count, C7520)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_mma<kBf16, kN>(acc, desc_lohi(a_lo + 2 * k, ab_hi), desc_lohi(b_lo + 2 * k, ab_hi), it != 0 || k != 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_s >= 0 && wg_leader) mbar_arrive(&empty_bar[team][prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      fence_acc<kN / 2>(acc);
      if (wg_leader) mbar_arrive(&empty_bar[team][prev_s]);
    }

#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      fr.row[rr] = static_cast<long long>(m0) + fr.loc[rr];
      fr.ok[rr] = fr.row[rr] < p.M;
    }
    // box b of the tile stays in the team's staging buffer b until the tail GEMM has read it, so the team's previous
    // stores must have drained both buffers before this tile writes them
    if (issuer) tma_store_wait_read<0>();
    named_bar_sync(team_bar, 256);
#pragma unroll
    for (int c0 = 0; c0 < kN; c0 += 64) {
      uint8_t* buf = team_staging + (c0 / 64) * kStageBufBytes;
      epilogue_box<kBf16, kN>(p.ep, acc, c0, 64, s_bias, fr, 0, buf, lane);
      fence_proxy_async_smem();
      named_bar_sync(team_bar, 256);
      if (issuer) {
        if (p.ch.store_first && c0 < p.ep.Cout) tma_store_2d(&tmap_out, buf, c0, m0);
        tma_store_commit();
      }
    }
    {
      // every box of the tile is in shared memory and visible to the async proxy (fence + barrier above)
      const uint32_t a2_hi = desc_hi(128, 8 * 128);
      const uint32_t w2_hi = desc_hi(p.ch.w2_row_bytes, 8 * p.ch.w2_row_bytes);
      const uint32_t stag_lo = smem_lo16(team_staging) + ((64 * half * 128) >> 4);
      const uint32_t w2_lo0 = smem_lo16(w2_res);
      const uint32_t w2_step16 = p.ch.w2_sub_bytes >> 4;
      wgmma_fence();
      // one or two 64-channel boxes feed the tail (conv_team_plan); each branch issues a fixed count of K steps
      if (p.ch.own_chunks == 2) {
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_mma<kBf16, kN2>(acc, desc_lohi(stag_lo + j * (kStageBufBytes >> 4) + 2 * k, a2_hi),
                                  desc_lohi(w2_lo0 + j * w2_step16 + 2 * k, w2_hi), (j | k) != 0);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_mma<kBf16, kN2>(acc, desc_lohi(stag_lo + 2 * k, a2_hi), desc_lohi(w2_lo0 + 2 * k, w2_hi), k != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc<kN2 / 2>(acc);
    }
    // the tail's box reuses staging buffer 0: the operand boxes are dead (both warpgroups' tail GEMMs have completed),
    // but the stores of the first output may still be reading them
    if (issuer) tma_store_wait_read<0>();
    named_bar_sync(team_bar, 256);
    EpilogueParams ep2 = p.ch.ep2;
    ep2.residual = nullptr;   // never set for a tail (chain_setup); known here, the epilogue drops its row addresses
#pragma unroll
    for (int c0 = 0; c0 < kN2; c0 += 64) {
      uint8_t* buf = team_staging + ((c0 / 64) & 1) * kStageBufBytes;
      epilogue_box<kBf16, kN2>(ep2, acc, c0, 64, s_bias2, fr, 0, buf, lane);
      fence_proxy_async_smem();
      if (issuer) tma_store_wait_read<0>();   // box k + 1 overwrites the buffer of box k - 1
      named_bar_sync(team_bar, 256);
      if (issuer) {
        if (c0 < p.ch.ep2.Cout) tma_store_2d(&tmap_out2, buf, c0, m0);
        tma_store_commit();
      }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

// ===================== four consumer warpgroups: two tiles per streamed weight slab =====================
// The deep 1x1 and stride-2 im2col launches whose weights do not fit in shared memory stream a 16 KB weight slab from L2
// for every k-iteration of every 128-row tile: as many bytes as their activations.  Here a task is two consecutive
// 128-row M tiles (2q, 2q + 1) x one 128-column N tile, and a pipeline stage holds both tiles' A sub-tiles and ONE
// weight slab, so the weight stream from L2 is halved.  Warpgroups 2t + 1 and 2t + 2 form team t, which owns tile t of
// the task as the two consumer warpgroups of conv_wgmma_kernel own a tile: 64 rows each, m64n128k16, 64 accumulators
// per thread.  All four read the slab; a stage is released (four arrivals) once the commit group after it completes.
// Per team: a named barrier (2 + t), two 16 KB staging boxes and a TMA-store issuer, so both teams' epilogues run while
// the producer fills the next task's stages.  Every output element gets the k16 MMA sequence and the epilogue of
// conv_wgmma_kernel, so the outputs are the same bits.  Only what these launches need is compiled: modes 0 and 1, whole
// 64-channel K chunks, streamed weights, 128 columns, one N tile per CTA (the grid is a multiple of the N tiles), no
// residual, chained tail, fused decode or split tail (conv_quad_plan).
constexpr size_t kQuadStaticSmem = 2 * kMaxStages * 8 + 128 * 4;   // barriers + bias vector (ptxas -v)
constexpr size_t kQuadSmemBudget = 227 * 1024 - kQuadStaticSmem;
constexpr int kQuadMinMTiles = 100;    // conv_quad_plan
constexpr int kQuadWideMTiles = 400;

template <bool kBf16>
__global__ void __launch_bounds__(kTeamThreads, 1)
conv_wgmma_quad_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap,
                       const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap,
                       const __grid_constant__ CUtensorMap, const ConvKernelParams p) {
  constexpr int kN = 128;
  constexpr int kStageBufBytes = stage_buf_bytes(2);
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ __align__(16) float s_bias[kN];

  uint8_t* tiles = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  // stage = [A of tile 0][A of tile 1][B slab]
  const uint32_t stage_bytes = 2 * p.a_stage_bytes + p.b_stage_bytes;
  uint8_t* staging = tiles + static_cast<size_t>(p.stages) * stage_bytes;   // [2 teams][kStageBufs][kStageBufBytes]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);   // every consumer warpgroup reads every stage
    }
    mbar_fence_init();
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // 128 x 24 + 512 x 112 <= 640 x 96: the producers lower their budget and return before the consumers raise theirs
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (warp != 0) return;
    // ===================== TMA producer: both tiles' A and one weight slab per k-iteration =====================
    const uint32_t a_bytes = p.a_stage_bytes, b_bytes = p.block_n * p.block_k * 2;
    const int m_tiles = p.num_tiles / p.n_tiles;
    int kit = 0;
    for (int t = blockIdx.x; t < p.num_tasks; t += gridDim.x) {
      const int q = t / p.n_tiles;
      const int n0 = (t - q * p.n_tiles) * p.block_n;
      const int cnt = min(2, m_tiles - 2 * q);   // the odd last pair has one tile
      for (int it = 0; it < p.num_k_iters; ++it, ++kit) {
        const int s = kit % p.stages;
        mbar_wait(&empty_bar[s], ((kit / p.stages) & 1) ^ 1);
        uint8_t* a_dst = tiles + s * stage_bytes;
        if (YB_ELECT()) {
          mbar_expect_tx(&full_bar[s], cnt * a_bytes + b_bytes);
          const int tap = it / p.chunks;
          const int chunk = it - tap * p.chunks;
          for (int j = 0; j < cnt; ++j) {
            const int m0 = (2 * q + j) * 128;
            if (p.mode == 0) {
              tma_load_2d(&tmap_a, &full_bar[s], a_dst + j * a_bytes, chunk * p.block_k, m0);
            } else {   // the tile's first output pixel, as conv_wgmma_kernel's producer derives it
              const int cn = m0 / p.HoWo;
              const int rem = m0 - cn * p.HoWo;
              const int ho = rem / p.Wo;
              const int wo = rem - ho * p.Wo;
              const int r = tap / p.ksize;
              const int sx = tap - r * p.ksize;
              tma_load_im2col_4d(&tmap_a, &full_bar[s], a_dst + j * a_bytes, chunk * p.block_k, wo * p.stride - p.pad,
                                 ho * p.stride - p.pad, cn, static_cast<uint16_t>(sx), static_cast<uint16_t>(r));
            }
          }
          tma_load_2d(&tmap_b, &full_bar[s], a_dst + 2 * a_bytes, it * p.block_k, n0);
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 112;\n" ::: "memory");

  // ===================== consumers: team `team`, warpgroup `half` of it multiplies rows 64 half .. +63 =====================
  const int cw = (warp >> 2) - 1;
  const int team = cw >> 1, half = cw & 1;
  const int wq = warp & 3;
  const int ctid = threadIdx.x - 128;
  const bool issuer = (ctid & 255) == 0;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint32_t team_bar = kTeamBar0 + team;
  FragRows fr;
  fr.loc[0] = half * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  uint8_t* team_staging = staging + static_cast<size_t>(team) * kStageBufs * kStageBufBytes;
  EpilogueParams ep = p.ep;
  ep.residual = nullptr;   // never set for these launches (conv_quad_plan); known here, the epilogue drops its row addresses
  float acc[kN / 2];

  // grid % n_tiles == 0 (conv_quad_plan): task % n_tiles, the N tile, is the same for every task of this CTA
  const int n0 = (blockIdx.x % p.n_tiles) * kN;
  for (int i = ctid; i < kN; i += 512) s_bias[i] = (n0 + i < p.bias_len) ? __ldg(p.bias + n0 + i) : 0.f;
  named_bar_sync(kConsumerBar, 512);

  const int m_tiles = p.num_tiles / p.n_tiles;
  int kit = 0, store_idx = 0;
  for (int t = blockIdx.x; t < p.num_tasks; t += gridDim.x) {
    const int mt = 2 * (t / p.n_tiles) + team;
    // Team 1 has no tile in the odd last pair.  It still issues its MMAs, on whatever its A slots hold, and discards the
    // result: a branch around the MMAs would make ptxas serialise every wgmma of the kernel (C7520).  It waits for and
    // releases every stage like the other warpgroups.
    const bool active = mt < m_tiles;
    const int m0 = mt * 128;
    {
      // descriptor constants, derived per task rather than held through the epilogue (registers are short)
      const uint32_t ab_hi = desc_hi(128, 8 * 128);                              // 64-channel rows of 128 bytes
      const uint32_t a_off16 = (p.a_stage_bytes * team + 64 * 128 * half) >> 4;   // this warpgroup's 64 rows
      const uint32_t b_off16 = (2 * p.a_stage_bytes) >> 4;
      const uint32_t tiles_lo = smem_lo16(tiles);
      const uint32_t stage16 = stage_bytes >> 4;
      // The first MMA overwrites the accumulators; zeroing them first tells ptxas that the previous task's values are
      // dead, which it cannot see through the run-time accumulate flag.
#pragma unroll
      for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
      // ---- main loop: stage s is released once the MMAs that read it have completed (one stage in flight) ----
      int prev_s = -1;
      for (int it = 0; it < p.num_k_iters; ++it, ++kit) {
        const int s = kit % p.stages;
        mbar_wait(&full_bar[s], (kit / p.stages) & 1);
        const uint32_t st_lo = tiles_lo + s * stage16;
        wgmma_fence();
        // whole 64-channel chunks (conv_quad_plan): four K steps, a fixed count (ptxas serialises the wgmmas of a
        // run-time count, C7520)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_mma<kBf16, kN>(acc, desc_lohi(st_lo + a_off16 + 2 * k, ab_hi), desc_lohi(st_lo + b_off16 + 2 * k, ab_hi),
                               it != 0 || k != 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_s >= 0 && wg_leader) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      fence_acc<kN / 2>(acc);
      if (wg_leader) mbar_arrive(&empty_bar[prev_s]);
    }

#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      fr.row[rr] = static_cast<long long>(m0) + fr.loc[rr];
      fr.ok[rr] = active && fr.row[rr] < p.M;
    }
    // the team's tile in two 64-column boxes through its two staging buffers: before the barrier the issuer waits until
    // the previous store has read its buffer, which the next box overwrites
#pragma unroll
    for (int c0 = 0; c0 < kN; c0 += 64, ++store_idx) {
      uint8_t* buf = team_staging + (store_idx & 1) * kStageBufBytes;
      epilogue_box<kBf16, kN>(ep, acc, c0, 64, s_bias, fr, n0, buf, lane);
      fence_proxy_async_smem();
      if (issuer) tma_store_wait_read<0>();
      named_bar_sync(team_bar, 256);
      if (issuer) {
        if (active && n0 + c0 < p.ep.Cout) tma_store_2d(&tmap_out, buf, n0 + c0, m0);
        tma_store_commit();
      }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

using ConvKernelFn =void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                              const CUtensorMap, const CUtensorMap, const ConvKernelParams);

// One kernel per (dtype, N tile, fused decode, chained tail N, CTAs per SM, consumer warpgroups): the MMA width and the
// accumulator size are compile-time constants of every instance, so the accumulators stay in registers while the wgmma
// instructions are in flight.  conv_configure admits exactly these shapes.
template <bool kBf16>
ConvKernelFn select_conv_kernel_t(const ConvKernelParams& kp) {
  if (kp.groups == 4 && kp.pair == 2)   // two-tile tasks over one streamed weight slab (conv_quad_plan)
    return kp.block_n == 128 && !kp.ch.on ? conv_wgmma_quad_kernel<kBf16> : nullptr;
  if (kp.groups == 4)   // two consumer teams (conv_team_plan): N = 128 with a 64-column tail
    return kp.block_n == 128 && kp.ch.n2 == 64 ? conv_wgmma_team_kernel<kBf16, 128, 64> : nullptr;
  if (kp.groups == 1) {
    // one consumer warpgroup, two CTAs per SM, at the one-CTA instances' 232 consumer registers: the 256-column layers,
    // as two 128-column N tiles (conv_plan).  No N = 256 instance: ptxas allocates against the 128 registers of
    // __launch_bounds__(256, 2), and one m64n256 wgmma needs 128 accumulators plus its operands.
    if (kp.ctas != 2 || kp.decode_on || kp.ch.on) return nullptr;
    return kp.block_n == 128 ? conv_wgmma_kernel<kBf16, 128, false, 0, 2, 1> : nullptr;
  }
  if (kp.ctas == 2) {
    // two CTAs per SM: the instances whose consumers fit in 104 registers without spilling (N <= 64, tails of at most
    // 64 columns; DESIGN.md section 3)
    if (kp.decode_on) return nullptr;
    if (kp.ch.on) {
      if (kp.block_n != 64) return nullptr;
      return kp.ch.n2 == 32 ? conv_wgmma_kernel<kBf16, 64, false, 32, 2>
                            : (kp.ch.n2 == 64 ? conv_wgmma_kernel<kBf16, 64, false, 64, 2> : nullptr);
    }
    switch (kp.block_n) {
      case 16: return conv_wgmma_kernel<kBf16, 16, false, 0, 2>;
      case 32: return conv_wgmma_kernel<kBf16, 32, false, 0, 2>;
      case 64: return conv_wgmma_kernel<kBf16, 64, false, 0, 2>;
      default: return nullptr;
    }
  }
  if (kp.decode_on) return conv_wgmma_kernel<kBf16, 256, true, 0, 1>;
  if (kp.ch.on) {
    if (kp.block_n == 64)
      return kp.ch.n2 == 32 ? conv_wgmma_kernel<kBf16, 64, false, 32, 1>
                            : (kp.ch.n2 == 64 ? conv_wgmma_kernel<kBf16, 64, false, 64, 1> : conv_wgmma_kernel<kBf16, 64, false, 128, 1>);
    return kp.ch.n2 == 32 ? conv_wgmma_kernel<kBf16, 128, false, 32, 1>
                          : (kp.ch.n2 == 64 ? conv_wgmma_kernel<kBf16, 128, false, 64, 1> : conv_wgmma_kernel<kBf16, 128, false, 128, 1>);
  }
  switch (kp.block_n) {
    case 16: return conv_wgmma_kernel<kBf16, 16, false, 0, 1>;
    case 32: return conv_wgmma_kernel<kBf16, 32, false, 0, 1>;
    case 64: return conv_wgmma_kernel<kBf16, 64, false, 0, 1>;
    case 128: return conv_wgmma_kernel<kBf16, 128, false, 0, 1>;
    default: return conv_wgmma_kernel<kBf16, 256, false, 0, 1>;
  }
}
ConvKernelFn select_conv_kernel(const ConvKernelParams& kp) {
  return kp.ep.is_bf16 ? select_conv_kernel_t<true>(kp) : select_conv_kernel_t<false>(kp);
}

}  // namespace

static int conv_plan(const yb_op_desc& d, int ctas, int groups, ConvKernelParams& kp, dim3& grid, size_t& smem_bytes);
static void conv_team_plan(ConvKernelParams& kp, size_t& smem_bytes);
static void conv_quad_plan(ConvKernelParams& kp, dim3& grid, size_t& smem_bytes);

// Validation of an fp16 / bf16 convolution descriptor, shared with the halo-patch kernel (pure host logic).
int conv_validate(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "conv: dtype must be f16 or bf16");
  YB_REQUIRE((d.reserved & ~(31 | YB_CONV_NO_TAIL_SPLIT | YB_CONV_PAIR_N64 | YB_CONV_NO_TEAMS)) == 0,
             "conv: reserved bits 5 and 9 and up must be zero, got 0x%x",
             d.reserved);
  YB_REQUIRE(d.ksize >= 1 && d.ksize <= 7 && d.stride >= 1 && d.stride <= 2, "conv: ksize/stride");
  YB_REQUIRE(d.act >= YB_ACT_NONE && d.act <= YB_ACT_RELU, "conv: unknown activation %d", d.act);
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
  int M;
  return conv_rows(d, "conv", &M);
}

// Pure host logic: validates the op and derives tiling, pipeline depth, shared-memory layout and launch shape
// (no driver calls: yb_conv_chain_supported runs this without a GPU).
static int conv_configure(const yb_op_desc& d, ConvKernelParams& kp, dim3& grid, size_t& smem_bytes) {
  const int rc = conv_validate(d);
  if (rc != YB_OK) return rc;
  YB_REQUIRE(!(d.reserved & YB_CONV_BAND_STEM),
             "conv: banded stem weights (reserved bit 1) need the halo-patch kernel, which this %dx%d map does not qualify for",
             d.H, d.W);
  // Five layouts, tried in this order:
  //   two CTAs of two consumer warpgroups (104 registers) when the shape has such an instance;
  //   otherwise two CTAs of ONE consumer warpgroup (64-row tiles, 232 registers) when the shape has that instance;
  //   otherwise one CTA of two consumer teams of two warpgroups when the one-CTA plan qualifies (conv_team_plan);
  //   otherwise one CTA of four consumer warpgroups on two-tile tasks when the one-CTA plan qualifies (conv_quad_plan);
  //   one CTA of two consumer warpgroups.
  // Each two-CTA plan must fit half of the SM's shared memory and have a tile for each of the 2 x SMs CTAs.
  // YB_CONV_ONE_CTA keeps the last layout (tests compare the launches bit for bit), and so does YB_CONV_PAIR_N64, which
  // names the two-warpgroup launch of every four-warpgroup one.  YB_CONV_NO_TEAMS keeps it instead of two teams, and
  // YB_CONV_NO_TAIL_SPLIT instead of two-tile tasks (its plan is the one-CTA plan of whole single tiles).
  if (!(d.reserved & YB_CONV_ONE_CTA) &&
      (conv_plan(d, 2, 2, kp, grid, smem_bytes) == YB_OK || conv_plan(d, 2, 1, kp, grid, smem_bytes) == YB_OK))
    return YB_OK;
  const int rc1 = conv_plan(d, 1, 2, kp, grid, smem_bytes);
  if (rc1 == YB_OK && !(d.reserved & (YB_CONV_ONE_CTA | YB_CONV_NO_TEAMS | YB_CONV_PAIR_N64)))
    conv_team_plan(kp, smem_bytes);
  if (rc1 == YB_OK && !(d.reserved & (YB_CONV_ONE_CTA | YB_CONV_PAIR_N64 | YB_CONV_NO_TAIL_SPLIT)))
    conv_quad_plan(kp, grid, smem_bytes);
  return rc1;
}

// Two consumer teams (conv_wgmma_team_kernel) for a one-CTA plan of a chained 1x1 / s1 launch (mode 0) with resident
// weights in one N tile of 128 columns, whole 64-channel K chunks, a 64-column tail over one or two 64-channel boxes and
// no fused decode -- the shapes the team instances compile -- when it has at least kTeamMinTilesPerSm tiles per SM and
// the weights, the tail weights, each team's two staging boxes and a ring of at least two 16 KB A stages per team fit
// in 227 KB less the kernel's static shared memory.  The tiling, the grid and the MMA sequence of every output element
// stay those of the one-CTA plan; only the A ring changes (one k-iteration per stage, one ring per team).  The
// threshold keeps every smaller launch on two warpgroups (DESIGN.md section 3).
static void conv_team_plan(ConvKernelParams& kp, size_t& smem_bytes) {
  if (!(kp.ctas == 1 && kp.groups == 2 && kp.mode == 0 && kp.ch.on && !kp.decode_on && kp.b_resident &&
        kp.n_tiles == 1 && kp.block_n == 128 && kp.ch.n2 == 64 && kp.block_k == 64 && kp.kk_last == 4 &&
        kp.ch.ksteps == 4 && kp.num_tiles >= kTeamMinTilesPerSm * num_sms()))
    return;
  const size_t fixed = kp.b_res_bytes + 2 * kStageBufs * static_cast<size_t>(stage_buf_bytes(2)) +
                       static_cast<size_t>(kp.ch.w2_chunks) * kp.ch.w2_sub_bytes + 1024;
  if (fixed >= kTeamSmemBudget) return;
  int stages = static_cast<int>((kTeamSmemBudget - fixed) / (2 * static_cast<size_t>(kp.a_stage_bytes)));
  if (stages < 2) return;
  if (stages > kTeamMaxStages) stages = kTeamMaxStages;
  kp.groups = 4;
  kp.kpg = 1;
  kp.stages = stages;
  smem_bytes = fixed + 2 * static_cast<size_t>(stages) * kp.a_stage_bytes;
}

// Two-tile tasks on four consumer warpgroups (conv_wgmma_quad_kernel) for a one-CTA plan that streams its weights in
// 128-column N tiles over whole 64-channel K chunks, without a residual, chained tail or fused decode -- the shapes the
// quad instances compile.  The T = ceil(m_tiles / 2) x n_tiles pair tasks run on G = min(T, SMs) CTAs, G a multiple of
// the N tiles (every CTA keeps one N tile).  These launches are bound by the L2 -> SM stream, which the shared weight
// slab cuts by a quarter, so they win even where the wider tasks add a round of the grid (c2's ops 8 and 27, 3.03
// rounds of pairs: DESIGN.md section 3).  The rule takes the sizes measured: at least kQuadMinMTiles M tiles, and
// either at most one per SM, three or more N tiles, or at least kQuadWideMTiles M tiles; other sizes keep two
// warpgroups (not measured).  The plan also needs two stages of two A sub-tiles and one weight slab next to both teams' staging boxes
// in 227 KB less the kernel's static shared memory.  The tiling and the MMA sequence of every output element stay
// those of the one-CTA plan; the task list, the grid and the pipeline change, and the split tail goes.
static void conv_quad_plan(ConvKernelParams& kp, dim3& grid, size_t& smem_bytes) {
  if (!(kp.ctas == 1 && kp.groups == 2 && !kp.b_resident && kp.block_n == 128 && !kp.ch.on && !kp.decode_on &&
        kp.ep.residual == nullptr && kp.block_k == 64 && kp.kk_last == 4))
    return;
  const int sms = num_sms();
  const int m_tiles = kp.num_tiles / kp.n_tiles;
  const int T = (m_tiles + 1) / 2 * kp.n_tiles;
  const int G = T < sms ? T : sms;
  if (G % kp.n_tiles != 0 || m_tiles < kQuadMinMTiles ||
      !(m_tiles <= sms || kp.n_tiles >= 3 || m_tiles >= kQuadWideMTiles))
    return;
  const uint32_t stage_bytes = 2 * kp.a_stage_bytes + kp.b_stage_bytes;
  const size_t fixed = 2 * kStageBufs * static_cast<size_t>(stage_buf_bytes(2)) + 1024;
  int stages = static_cast<int>((kQuadSmemBudget - fixed) / stage_bytes);
  if (stages < 2) return;
  if (stages > kMaxStages) stages = kMaxStages;
  kp.groups = 4;
  kp.pair = 2;
  kp.kpg = 1;
  kp.stages = stages;
  kp.split = 1;
  kp.full_tiles = kp.num_tiles;
  kp.num_tasks = T;
  grid = dim3(G, 1, 1);
  smem_bytes = fixed + static_cast<size_t>(stages) * stage_bytes;
}

// Tiling, pipeline depth, shared-memory layout and launch shape for `ctas` CTAs per SM of `groups` consumer warpgroups
// (conv_configure has validated the descriptor).  With ctas = 2 the plan gets half of the SM's shared memory, less the
// per-CTA reservation and the kernel's static shared memory, and fails when it does not fit there, when the layout has
// no instance for the shape or when there are fewer tiles than 2 x SMs.  One consumer warpgroup is only planned for
// shapes without a 104-register two-CTA instance.
static int conv_plan(const yb_op_desc& d, int ctas, int groups, ConvKernelParams& kp, dim3& grid, size_t& smem_bytes) {
  const int Ho = d.Ho, Wo = d.Wo;
  const size_t budget = ctas == 2 ? smem_per_sm() / 2 - kSmemReservedPerCta - kStaticSmem : kSmemBudget;
  const int block_m = tile_rows(groups);
  kp = ConvKernelParams();
  kp.ctas = ctas;
  kp.groups = groups;
  kp.pair = 1;
  kp.M = static_cast<int>(static_cast<long long>(d.N) * Ho * Wo);
  kp.ep.Cout = d.Cout;
  const int m_tiles = (kp.M + block_m - 1) / block_m;
  const int sms = num_sms();
  const int m_tiles128 = (kp.M + tile_rows(2) - 1) / tile_rows(2);
  int block_n = conv_block_n(d.Cout, m_tiles128, d.chain != nullptr);   // the same N tile in every layout
  if (groups == 1) {
    // one consumer warpgroup: only layers whose one-CTA plan has a 256-column N tile, split into two 128-column ones,
    // with at least 3 x SMs 128-row tiles (DESIGN.md section 3: measured gains at 400 and 1600 such tiles, none at 100)
    if (block_n != 256 || d.chain != nullptr || m_tiles128 < 3 * sms) return YB_ERR_INVALID;
    block_n = 128;
  }
  // A one-CTA 256-column plan that streams its weights (more than 80 KB) and runs 2-4 rounds, the last one partial,
  // takes 128-column N tiles instead when the split tail then applies (see below): with so few rounds the idle part of
  // the last one is a large share of the launch.  c2's ops 8 and 27 (3.03 rounds) measured 145 -> 114 and 106 -> 73 us;
  // launches with more rounds keep 256 columns (not measured).
  // The bits that pin a plan for bit-for-bit comparisons (YB_CONV_ONE_CTA, YB_CONV_NO_TAIL_SPLIT) keep 256 columns.
  if (groups == 2 && ctas == 1 && block_n == 256 && d.chain == nullptr && d.decode == nullptr &&
      !(d.reserved & (YB_CONV_NO_TAIL_SPLIT | YB_CONV_ONE_CTA)) && static_cast<size_t>(d.ksize) * d.ksize * d.Cin_pad * 256 * 2 > 80 * 1024 &&
      m_tiles > sms && m_tiles < 4 * sms && m_tiles % sms != 0) {
    const int n128 = (d.Cout + 127) / 128, r128 = (m_tiles * n128) % sms;
    if (sms % n128 == 0 && r128 > 0 && 2 * r128 <= sms) block_n = 128;
  }
  int n_tiles = (d.Cout + block_n - 1) / block_n;
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
  kp.a_stage_bytes = block_m * kp.block_k * 2;
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
  // A one-group plan (grid 2 x SMs) also keeps the weights resident over several N tiles when the grid is a multiple of
  // the N tiles: every CTA then has one N tile and holds its weights.
  const size_t fixed = static_cast<size_t>(kStageBufs) * stage_buf_bytes(groups) + 1024 + chain_bytes;
  const bool fixed_n = n_tiles == 1 || (groups == 1 && (2 * sms) % n_tiles == 0);
  KPipeline pipe;
  const int rc = size_k_pipeline(budget, fixed, kp.a_stage_bytes, kp.b_stage_bytes, kp.num_k_iters, fixed_n, kMaxStages,
                                 "conv", kp.block_n, &pipe);
  if (rc != YB_OK) return rc;
  kp.b_resident = pipe.b_resident;
  kp.b_res_bytes = pipe.b_res_bytes;
  kp.kpg = pipe.kpg;
  kp.stages = pipe.stages;
  kp.ep.is_bf16 = d.dtype == YB_BF16;
  kp.ep.act = d.act;
  kp.bias = d.bias;
  kp.ep.residual = d.residual;
  kp.ep.res_cstride = d.res_cstride;
  // two CTAs per SM: only with an instance built for it and at least one tile for each of the 2 x SMs CTAs
  if (ctas == 2 && (select_conv_kernel(kp) == nullptr || kp.num_tiles < 2 * sms)) return YB_ERR_INVALID;
  if (groups == 1) {   // only with resident weights, and where the shape has no 104-register two-CTA instance
    ConvKernelParams two = kp;
    two.groups = 2;
    if (!kp.b_resident || select_conv_kernel(two) != nullptr) return YB_ERR_INVALID;
  }
  const int max_grid = ctas * sms;   // a grid that is not a multiple of the N tiles loads the bias per tile
  grid = dim3(kp.num_tiles < max_grid ? kp.num_tiles : max_grid, 1, 1);
  // Split tail: when the tiles are not a whole number of rounds of the grid, the r tiles of the last round would leave
  // G - r CTAs idle for a whole tile time.  With 128-column N tiles each of them becomes two sub-tasks, which the idle
  // CTAs run: 64-row halves (both warpgroups on the same 64 A rows, 64 columns each) with two consumer warpgroups,
  // 64-column halves with one.  Each warpgroup keeps the wgmma M of 64 rows and the k16 sequence, so every output
  // element is computed as in the whole tile and the results are bit-identical.  A last round fuller than G / 2 cannot
  // be halved within one round and stays.
  const int G = static_cast<int>(grid.x);
  const int r = kp.num_tiles % G;
  kp.split = !(d.reserved & YB_CONV_NO_TAIL_SPLIT) && !kp.decode_on && !kp.ch.on && kp.block_n == 128 &&
                     G % kp.n_tiles == 0 && r > 0 && 2 * r <= G ? 2 : 1;
  kp.full_tiles = kp.split > 1 ? kp.num_tiles - r : kp.num_tiles;
  kp.num_tasks = kp.full_tiles + (kp.num_tiles - kp.full_tiles) * kp.split;
  smem_bytes = pipe.smem;
  return YB_OK;
}

int im2col_conv_config(const yb_op_desc& d, yb_conv_info* info) {
  ConvKernelParams kp;
  dim3 grid;
  size_t smem = 0;
  const int rc = conv_configure(d, kp, grid, smem);
  if (rc == YB_OK && info) {   // yb_conv_config: see include/yolort_b200.h
    info->kernel = YB_CONV_KERNEL_IM2COL;
    info->block_n = kp.block_n;
    info->n_tiles = kp.n_tiles;
    info->weights_resident = kp.b_resident;
    info->tiles_per_pass = kp.pair;
    info->slots = kp.stages;
    info->ring = kp.kpg;
    info->store_cols = kp.store_cols;
    info->store_bufs = kStageBufs;   // shared by the consumer warpgroups (of a team, with two teams)
    info->groups = kp.groups;
    info->resident_ctas = kp.ctas;
    info->chained = kp.ch.on;
    info->smem_bytes = static_cast<int>(smem);
    info->grid = static_cast<int>(grid.x);
    info->tiling = YB_CONV_TILING_ROWS;
    info->m_tiles = kp.num_tiles / kp.n_tiles;
    info->work_items = kp.num_tiles;
    info->tail_n = kp.ch.n2;
    info->tail_tiles = kp.split > 1 ? kp.num_tiles - kp.full_tiles : 0;
    info->tail_split = kp.split;
  }
  return rc;
}

struct Im2colConvOp final : ConvOp {
  CUtensorMap tmap_a, tmap_b, tmap_out, tmap_w2, tmap_out2, tmap_a64, tmap_out64;
  ConvKernelParams kp;
  ConvKernelFn fn = nullptr;
  dim3 grid;
  size_t smem_bytes;
  int launch(cudaStream_t stream) const override {
    YB_CHECK_CUDA(launch_pdl(fn, grid, dim3(cta_threads(kp.groups)), smem_bytes, stream, tmap_a, tmap_b, tmap_out, tmap_w2,
                             tmap_out2, tmap_a64, tmap_out64, kp));
    return YB_OK;
  }
};

int im2col_conv_create(const yb_op_desc& d, ConvOp** out) {
  Im2colConvOp* op = new Im2colConvOp();
  ConvKernelParams& kp = op->kp;
  int rc = conv_configure(d, kp, op->grid, op->smem_bytes);
  const bool teams = kp.groups == 4;   // two consumer teams, or two-tile tasks on four consumer warpgroups
  const uint32_t block_m = tile_rows(teams ? 2 : kp.groups);   // rows of the A, output and tail-output boxes
  const CUtensorMapDataType dt = kp.ep.is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  if (rc == YB_OK)
    rc = kp.mode == 0 ? tmap_matrix(&op->tmap_a, "conv input", dt, d.in, d.Cin, kp.M, d.in_cstride, kp.block_k, block_m,
                                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B)
                      : tmap_im2col(&op->tmap_a, "conv input", dt, d, kp.block_k, block_m);
  const int ktot = d.ksize * d.ksize * d.Cin_pad;
  if (rc == YB_OK)
    rc = tmap_matrix(&op->tmap_b, "conv weights", dt, d.weight, ktot, d.Cout_pad, ktot, kp.block_k, kp.block_n,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  // destination view [M rows, Cout channels], row pitch = out_cstride; boxes of block_m rows x store_cols
  if (rc == YB_OK)
    rc = tmap_matrix(&op->tmap_out, "conv output", dt, d.out, d.Cout, kp.M, d.out_cstride, kp.store_cols, block_m,
                     CU_TENSOR_MAP_L2_PROMOTION_NONE);
  op->tmap_w2 = op->tmap_b;      // placeholders when nothing is chained (never dereferenced)
  op->tmap_out2 = op->tmap_out;
  op->tmap_a64 = op->tmap_a;     // ... and when no tail tile is split into row halves
  op->tmap_out64 = op->tmap_out;
  if (rc == YB_OK && kp.split > 1 && kp.groups == 2) {   // the row halves' 64-row A and output boxes
    rc = kp.mode == 0 ? tmap_matrix(&op->tmap_a64, "conv input (tail halves)", dt, d.in, d.Cin, kp.M, d.in_cstride,
                                    kp.block_k, 64, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)
                      : tmap_im2col(&op->tmap_a64, "conv input (tail halves)", dt, d, kp.block_k, 64);
    if (rc == YB_OK)
      rc = tmap_matrix(&op->tmap_out64, "conv output (tail halves)", dt, d.out, d.Cout, kp.M, d.out_cstride, kp.store_cols,
                       64, CU_TENSOR_MAP_L2_PROMOTION_NONE);
  }
  if (rc == YB_OK && kp.ch.on) {
    const yb_conv_chain& c = *d.chain;
    rc = tmap_matrix(&op->tmap_w2, "conv chained tail weights", dt, c.weight, c.K_pad, c.Cout_pad, c.K_pad,
                     kp.ch.w2_row_bytes / 2, kp.ch.n2, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc == YB_OK)
      rc = tmap_matrix(&op->tmap_out2, "conv chained tail output", dt, c.out, c.Cout, kp.M, c.out_cstride,
                       chain_store2_cols(kp.ch.n2), block_m, CU_TENSOR_MAP_L2_PROMOTION_NONE);
  }
  if (rc == YB_OK) {
    op->fn = select_conv_kernel(kp);
    const size_t budget = kp.pair == 2 ? kQuadSmemBudget : (teams ? kTeamSmemBudget : kSmemBudget);
    rc = set_smem_attributes(reinterpret_cast<const void*>(op->fn), budget, kp.ctas, op->smem_bytes,
                             cta_threads(kp.groups), "conv");
    if (rc == YB_OK && teams) {   // the 640-thread CTA with up to 227 KB of shared memory must fit on an SM
      int per_sm = 0;
      const cudaError_t e =
          cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, op->fn, cta_threads(kp.groups), op->smem_bytes);
      if (e != cudaSuccess) {
        set_error("conv: cudaOccupancyMaxActiveBlocksPerMultiprocessor failed: %s", cudaGetErrorString(e));
        rc = YB_ERR_CUDA;
      } else if (per_sm < 1) {
        set_error("conv: the four-warpgroup CTA (%d threads, %zu bytes of shared memory) does not fit on an SM",
                  cta_threads(kp.groups), op->smem_bytes);
        rc = YB_ERR_INVALID;
      }
    }
  }
  if (rc != YB_OK) {
    delete op;
    return rc;
  }
  *out = op;
  return YB_OK;
}

}  // namespace yb
