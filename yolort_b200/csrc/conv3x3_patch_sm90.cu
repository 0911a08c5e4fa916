// 3x3 / stride 1 / pad 1 convolution with the input halo patch staged ONCE per output tile.
//
// Why a second kernel: with im2col tensor maps every filter tap re-fetches its 128 pixels, i.e. the SM ingests 9x the
// tile's input (plus the weights) through the TMA path.  Here an output tile is a 16 x 8 pixel block of one image; its
// (16+2) x (8+2) input halo is fetched by ONE tiled 4-D TMA load per 64-channel chunk (box 18 x 10 pixels, halo
// zero-filled by the TMA unit), and the nine filter taps are nine *views* of that patch: tap (dy,dx) starts
// (dy*10 + dx) pixel-rows into the patch, rows of one 8-pixel group are contiguous and consecutive groups are exactly
// one patch row (10 pixel-rows) apart, which is what a K-major wgmma shared-memory descriptor expresses (SBO = 10 *
// row_bytes; the swizzle phase follows the absolute shared-memory address, so a view may start inside a swizzle atom).
// Input traffic per tile drops from 9 x 128 to 180 pixel-rows (6.4x less).
//
// Same arithmetic as conv_sm90.cu (yolort/v5/models/common.py:42-73,94-116): BN folded, bias + SiLU (+ residual)
// epilogue, fp32 accumulation.
//
// Stride 2 (the down-sampling convolutions body.1/3/5/7 and the two of the PAN): the input is split by COLUMN PARITY
// into two planes -- a 5-D tensor map [C, parity, W/2, H, N] over the same NHWC memory, no copy -- and one TMA box per
// plane fetches a 33 x 9 patch (33 input rows, pair-columns x0-1 .. x0+7).  Filter column dx = 0 is the odd plane one
// pair-column to the left, dx = 1 the even plane, dx = 2 the odd plane; consecutive output pixels are consecutive
// pair-columns (rows of a view stay contiguous) and consecutive output rows are two patch rows apart (SBO = 18 rows).
//
// Roles (one persistent CTA per SM, two for the narrow shallow levels, see patch_conv_configure; 384 threads): warp 0 = patch (A) producer, warp 2 = weight (B) producer (unless
// the weights are resident in shared memory), warpgroups 1-2 = consumers: each multiplies 64 of the tile's 128
// accumulator rows with wgmma (fp32 accumulators in registers) and runs the epilogue on its fragment.  Pair tasks with
// 128-column N tiles run on a lean instance of four consumer warpgroups (conv3x3_patch_quad_kernel, 640 threads).  The
// banded stem and the chains after a 64-column N tile, whose resident weights leave room for one CTA per SM only, run
// large launches on another 640-thread instance: two teams of two consumer warpgroups take the CTA's single-tile tasks
// alternately, so one team's epilogue and chained tail overlap the other team's MMAs (conv3x3_patch_team_kernel).
#include <cstdlib>

#include "common.cuh"
#include "conv_epilogue.cuh"
#include "conv_chain.cuh"
#include "conv_sm90.h"

namespace yb {
namespace {

constexpr int kMaxA = 4, kMaxB = 12;
constexpr int kConsumers = 2;                       // consumer warpgroups (64 accumulator rows each)
constexpr int kThreads = 128 * (1 + kConsumers);   // 384
constexpr int kStageBufBytes = 128 * 128;
constexpr int kMaxBlockN = 128;
constexpr size_t kSmemBudget = 216 * 1024;
constexpr size_t kStaticSmem = (2 * kMaxA + 2 * kMaxB + 2) * 8 + 2 * kMaxBlockN * 4;   // barriers + bias vectors (ptxas -v)
constexpr uint32_t kConsumerBar = 1;               // named barrier of the 256 consumer threads

// Tile geometry.  An output tile is 128 accumulator rows = 16 groups of 8 horizontally adjacent pixels.
//   classic: 16 rows x 8 columns (one group per tile row); patch 18 x 10, a tap view's groups are one patch row apart
//            (SBO = 10 pixel-rows).
//   wrap   : 5 rows x 24 columns for maps at most 22 pixels wide (the 20 x 20 level of a 640 canvas, which 16 x 8
//            tiles cover to 52 %): the patch pitch EQUALS the tile width (24 = x in [-1, 22]), so consecutive groups --
//            along a row and across rows -- are uniformly 8 pixel-rows apart and a tap view is one plain contiguous
//            128-row operand (SBO = 8 rows).  Rows 120..127 and columns >= W are junk that the TMA store clips.
struct TileGeom {
  int tile_h, tile_w;     // TMA store box (rows, columns); columns >= W are clipped by the store
  int x_step;             // output columns advanced per tile in x (classic 8; wrap: the whole width)
  int pitch, patch_h;     // patch = TMA load box: patch_h rows of `pitch` pixels, origin (x0 - 1, y0 - 1)
  int gpr;                // 8-pixel groups per tile row
  int sbo_rows;           // pixel-rows between consecutive groups of a tap view
  int alloc_rows;         // pixel-rows reserved per patch (>= what the junk rows of a view may touch)
};

struct PatchParams {
  int N, H, W;
  int tiles_x, tiles_y, m_tiles, n_tiles, num_tasks;
  int block_n, block_k, chunks;
  int a_slots, b_stages, b_resident;
  int pair;               // M tiles per weight pass: 2 = two patches share every weight slab (halves the L2 -> smem weight
                          // stream of the layers whose weights do not fit in shared memory); the consumers then hold
                          // the accumulators of both tiles (N tile <= 128)
  int s2;                 // 1: stride-2 convolution over two column-parity planes (H, W are the OUTPUT extent)
  int band;               // 1: banded super-pixel weights (stem), see the band MMA loop
  int ctas;               // CTAs per SM the launch is planned for (1 or 2): selects the kernel instance
  int teams;              // 1: two consumer teams of two warpgroups share the CTA (conv3x3_patch_team_kernel)
  int store_cols, store_bufs, bias_len;
  int stage_buf_bytes;    // bytes between the staging buffers (16 KB; 8 KB for the N-split variant)
  int kk_last;            // K=16 steps of the last channel chunk (TMA zero-fills past Cin, the MMA skips)
  TileGeom tg;
  uint32_t a_bytes, a_stride, b_sub_bytes, b_res_bytes;   // a_stride: bytes reserved per patch
  const float* bias;
  EpilogueParams ep;
  ChainParams ch;         // chained pointwise tail (kChain kernels; single-tile tasks with resident weights only)
};

__device__ __forceinline__ void tma_load_tiled_4d(const void* desc, uint64_t* bar, void* smem_dst, int c, int w,
                                                  int h, int n) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n)
      : "memory");
}
__device__ __forceinline__ void tma_load_tiled_5d(const void* desc, uint64_t* bar, void* smem_dst, int c, int par, int w,
                                                  int h, int n) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c), "r"(par), "r"(w), "r"(h), "r"(n)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* desc, const void* smem_src, int c, int w, int h, int n) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_u32(smem_src)), "r"(c), "r"(w), "r"(h), "r"(n)
               : "memory");
}

// (image, tile row, tile column) of an M tile
__device__ __forceinline__ void tile_coords(const PatchParams& p, int m_tile, int& n_img, int& y0, int& x0) {
  const int tpi = p.tiles_x * p.tiles_y;
  n_img = m_tile / tpi;
  const int t = m_tile - n_img * tpi;
  const int ty = t / p.tiles_x, tx = t - ty * p.tiles_x;
  y0 = ty * p.tg.tile_h;
  x0 = tx * p.tg.x_step;
}

__device__ __forceinline__ void consumer_sync() { named_bar_sync(kConsumerBar, 128 * kConsumers); }

// The K=16 steps of one filter tap over one channel chunk.
//   mode 0: one tile; 1: two tiles sharing the weight slab (second accumulator at acc + kN / 2, kPair instances only);
//   2: stride 2, one accumulator, the tap picks its column-parity plane (a0 = even plane, a1 = odd plane).
template <bool kBf16, int kN, bool kPair>
__device__ __forceinline__ void issue_tap(int mode, int tap, int kc, bool first, float* acc, uint32_t a0, uint32_t a1,
                                          uint32_t a_hi, uint32_t b_lo, uint32_t b_hi) {
  for (int k = 0; k < kc; ++k) {
    const bool accum = !(first && k == 0);
    const uint64_t db = desc_lohi(b_lo + 2 * k, b_hi);
    if (mode == 2) {
      wgmma_mma<kBf16, kN>(acc, desc_lohi(((tap % 3) == 1 ? a0 : a1) + 2 * k, a_hi), db, accum);
    } else {
      wgmma_mma<kBf16, kN>(acc, desc_lohi(a0 + 2 * k, a_hi), db, accum);
      if constexpr (kPair) {
        if (mode == 1) wgmma_mma<kBf16, kN>(acc + kN / 2, desc_lohi(a1 + 2 * k, a_hi), db, accum);
      }
    }
  }
}

// Epilogue of one M tile: boxes of store_cols columns through the staging buffers, TMA-stored as tile boxes.
template <bool kBf16, bool kChain, int kN>
__device__ __forceinline__ void store_tile(const PatchParams& p, const CUtensorMap* tmap_out, const float* acc, const float* s_bias,
                                           const FragRows& fr, int n0, int x0, int y0, int n_img, uint8_t* staging,
                                           int& store_idx, bool issuer, int lane) {
  const int store_cols = p.store_cols;
  for (int c0 = 0; c0 < p.block_n; c0 += store_cols, ++store_idx) {
    // Two staging buffers, one barrier per box: before the barrier below the issuer waits until the PREVIOUS store has
    // finished reading its buffer, which is the one the next box will overwrite.
    uint8_t* buf = staging + (kChain ? (c0 / store_cols) * kStageBufBytes : (p.store_bufs == 2 ? (store_idx & 1) * p.stage_buf_bytes : 0));
    if (!kChain && p.store_bufs == 1) {   // one staging buffer (stride-2 variant: the planes need the room): drain it first
      if (issuer) tma_store_wait_read<0>();
      consumer_sync();
    }
    epilogue_box<kBf16, kN>(p.ep, acc, c0, store_cols, s_bias, fr, n0, buf, lane);
    fence_proxy_async_smem();
    if constexpr (!kChain) {
      if (issuer && p.store_bufs == 2) tma_store_wait_read<0>();
    }
    consumer_sync();
    if (issuer) {
      if ((!kChain || p.ch.store_first) && n0 + c0 < p.ep.Cout) tma_store_4d(tmap_out, buf, n0 + c0, x0, y0, n_img);
      tma_store_commit();
    }
  }
}

// kN: the wgmma N of the tile (= block_n; pair tasks hold two tiles' accumulators, see kPair).  kN2 != 0: a pointwise
// tail of kN2 columns is chained onto every tile (conv_chain.cuh):
// tmap_w2 = its weights, tmap_x = its optional second operand block (C3: the cv2 half of the concat, fetched per tile
// with the output tile's box), tmap_out2 = its output.  kCtas: CTAs resident per SM (1 or 2, see regs_producer); with
// two, one CTA's epilogue and barrier waits overlap the other CTA's MMAs and patch loads.
template <bool kBf16, int kN, int kN2, int kCtas>
__global__ void __launch_bounds__(kThreads, kCtas)
conv3x3_patch_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_w2,
                     const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_out2,
                     const PatchParams p) {
  constexpr bool kChain = kN2 != 0;
  // Pair tasks (two tiles per weight pass) need the accumulators of two tiles: one-CTA instances with kN <= 64.  The
  // two-CTA instances only run single-tile tasks (patch_conv_plan) and hold one tile's accumulators.
  constexpr bool kPair = kCtas == 1 && kN <= 64;
  constexpr int kTileAcc = kPair ? kN : kN / 2;   // accumulator registers per thread
  // Two-CTA plans (patch_conv_plan) always have resident weights in one N tile, single-tile tasks and no banded stem:
  // those instances drop the other paths at compile time, which keeps their consumers within 104 registers.
  constexpr bool kLean = kCtas == 2;
  // Register budget.  The N = 128 instance and the N = 64 instances with a chained tail spill within the 168 registers
  // that __launch_bounds__ gives every thread, so their producers hand registers to the consumers (40 / 232).  The
  // other instances fit in 168 without spilling and keep the even split: with 232 registers ptxas builds a schedule for
  // them that runs 1-2.5 % slower on the H100 (pair-task and stride-2 launches).  With two CTAs per SM the even split
  // is 80 registers, too few for the consumers: every two-CTA instance takes the 24 / 104 split.
  constexpr bool kRealloc = kCtas == 2 || kN == 128 || (kChain && kN == 64);
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[kMaxA], a_empty[kMaxA];
  __shared__ __align__(8) uint64_t b_full[kMaxB], b_empty[kMaxB];
  __shared__ __align__(8) uint64_t x_full;    // chain: the extra operand block has landed
  __shared__ __align__(8) uint64_t w2_full;
  __shared__ __align__(16) float s_bias[kMaxBlockN];
  __shared__ __align__(16) float s_bias2[kChain ? kMaxBlockN : 4];

  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* a_buf = base;                                                      // [a_slots][a_stride]
  uint8_t* b_buf = a_buf + static_cast<size_t>(p.a_slots) * p.a_stride;        // resident [9*chunks] or ring [b_stages]
  const size_t b_region = p.b_resident ? p.b_res_bytes : static_cast<size_t>(p.b_stages) * p.b_sub_bytes;
  uint8_t* staging = b_buf + b_region;                                        // [store_bufs][stage_buf_bytes]
  uint8_t* w2_res = staging + static_cast<size_t>(p.store_bufs) * p.stage_buf_bytes;   // chain: tail weights

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int taps_total = 9 * p.chunks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < p.a_slots; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], kConsumers);   // one arrival per consumer warpgroup
    }
    for (int s = 0; s < kMaxB; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], kConsumers);
    }
    mbar_init(&x_full, 1);
    mbar_init(&w2_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above overlapped the tail of the previous kernel in the stream.  The
  // weight producer (warp 2) does not wait at all -- weights do not depend on the previous kernel, so the resident set
  // (or the first slabs of the ring) streams in while the previous kernel drains; every other warp touches activations
  // (or stores over them) and waits for the previous grid to complete first.
  if (warp != 2) asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // Each role raises or lowers its register budget on a path of its own: the producer warps return before the consumer
  // code, so ptxas never reaches the consumers from the 40-register budget.
  if constexpr (kRealloc) {
    if (warp < 4) regs_producer<kCtas>();
  }

  if (warp == 0) {
    // ===================== patch (A) producer (warp-uniform loop, one elected lane issues) =====================
    int ka = 0;   // patches issued so far (ring position)
    for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
      const int m_first = (task / p.n_tiles) * p.pair;
      const int cnt = p.s2 ? 2 : min(p.pair, p.m_tiles - m_first);   // patches per chunk: tiles of a pair, or the two planes
      for (int c = 0; c < p.chunks; ++c) {
        for (int j = 0; j < cnt; ++j, ++ka) {
          int n_img, y0, x0;
          tile_coords(p, p.s2 ? m_first : m_first + j, n_img, y0, x0);
          const int s = ka % p.a_slots;
          mbar_wait(&a_empty[s], ((ka / p.a_slots) & 1) ^ 1);
          if (YB_ELECT()) {
            mbar_expect_tx(&a_full[s], p.a_bytes);
            uint8_t* dst = a_buf + static_cast<size_t>(s) * p.a_stride;
            if (p.s2)   // plane j (0 = even columns, 1 = odd): pair-columns x0-1 .., input rows 2*y0-1 ..
              tma_load_tiled_5d(&tmap_a, &a_full[s], dst, c * p.block_k, j, x0 - 1, 2 * y0 - 1, n_img);
            else
              tma_load_tiled_4d(&tmap_a, &a_full[s], dst, c * p.block_k, x0 - 1, y0 - 1, n_img);
          }
        }
      }
    }
    return;
  }
  if (warp == 2) {
    // ===================== weight (B) producer =====================
    const uint32_t b_bytes = p.block_n * p.block_k * 2;
    if (p.band) {
      // banded stem weights: 3 filter rows x 2 blocks of 64 K-columns, consecutive in the weight matrix
      if (lane == 0) {
        mbar_expect_tx(&b_full[0], 6 * b_bytes);
        for (int i = 0; i < 6; ++i)
          tma_load_2d(&tmap_b, &b_full[0], b_buf + static_cast<size_t>(i) * p.b_sub_bytes, i * p.block_k, 0);
      }
    } else if (p.b_resident) {
      // With several N tiles the grid is a multiple of their count (host), so task % n_tiles -- the N tile -- is the
      // same for every task of this CTA: its slice of the weights stays resident.
      const int n0_res = (blockIdx.x % p.n_tiles) * p.block_n;
      if constexpr (kChain) {
        if (lane == 0) {   // tail weights: [n2][kc] chunks, resident for the CTA's lifetime
          tma_prefetch_desc(&tmap_w2);
          tma_prefetch_desc(&tmap_out2);
          if (p.ch.extra_on) tma_prefetch_desc(&tmap_x);
          mbar_expect_tx(&w2_full, p.ch.w2_chunks * p.ch.n2 * p.ch.w2_row_bytes);
          for (int j = 0; j < p.ch.w2_chunks; ++j)
            tma_load_2d(&tmap_w2, &w2_full, w2_res + j * p.ch.w2_sub_bytes, j * (p.ch.w2_row_bytes >> 1), 0);
        }
      }
      if (lane == 0) {
        mbar_expect_tx(&b_full[0], taps_total * b_bytes);
        for (int i = 0; i < taps_total; ++i)   // i = chunk*9 + tap ; weight column block = tap*chunks + chunk
          tma_load_2d(&tmap_b, &b_full[0], b_buf + static_cast<size_t>(i) * p.b_sub_bytes,
                      ((i % 9) * p.chunks + i / 9) * p.block_k, n0_res);
      }
    } else {
      int kb = 0;
      for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
        const int n0 = (task % p.n_tiles) * p.block_n;
        for (int i = 0; i < taps_total; ++i, ++kb) {
          const int s = kb % p.b_stages;
          mbar_wait(&b_empty[s], ((kb / p.b_stages) & 1) ^ 1);
          if (YB_ELECT()) {
            mbar_expect_tx(&b_full[s], b_bytes);
            tma_load_2d(&tmap_b, &b_full[s], b_buf + static_cast<size_t>(s) * p.b_sub_bytes,
                        ((i % 9) * p.chunks + i / 9) * p.block_k, n0);
          }
        }
      }
    }
    return;
  }
  if (warp < 4) return;
  if constexpr (kRealloc) regs_consumer<kCtas>();

  // ===================== consumers: MMA + epilogue of 64 accumulator rows each =====================
  const int g = (warp >> 2) - 1;
  const int wq = warp & 3;
  const bool issuer = threadIdx.x == 128;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int ctid = threadIdx.x - 128;
  const uint32_t row_bytes = p.block_k * 2;
  const int pitch = p.tg.pitch;   // pixel-rows per patch row
  const uint32_t sbo = p.tg.sbo_rows * row_bytes;
  const uint32_t a_wg16 = (8 * sbo * g) >> 4;   // this warpgroup's 64 rows: 8 groups of 8 further into every view
  const int kk = p.block_k >> 4;
  FragRows fr;
  fr.loc[0] = g * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  // position of this thread's accumulator rows inside a tile
  int yy[2], xx[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int grp = fr.loc[rr] >> 3;
    yy[rr] = grp / p.tg.gpr;
    xx[rr] = (grp - yy[rr] * p.tg.gpr) * 8 + (fr.loc[rr] & 7);
  }
  // per-tap start-address offsets of the A views (16-byte units) and the constant descriptor halves
  // tap (dy, dx) starts dy patch rows and dx pixel-rows into the patch (stride 2: dx = 0 reads the odd plane one
  // pair-column to the left of the output column, dx = 1 / 2 the even / odd plane at the output's own pair-column);
  // recomputed per tap rather than held in registers next to the accumulators
  const uint32_t row16 = row_bytes >> 4;
  auto tap_off16 = [&](int tap) -> uint32_t {
    const int dy = tap / 3, dx = tap - dy * 3;
    return static_cast<uint32_t>(dy * pitch + (p.s2 ? (dx == 0 ? 0 : 1) : dx)) * row16;
  };
  const uint32_t a_hi = desc_hi(row_bytes, sbo);
  const uint32_t b_hi = desc_hi(row_bytes, 8 * row_bytes);
  const uint32_t b_res_lo0 = smem_lo16(b_buf);
  const uint32_t b_step16 = p.b_sub_bytes >> 4;
  const int mode = p.s2 ? 2 : (p.pair == 2 ? 1 : 0);
  float acc[kTileAcc];

  if constexpr (kChain) {   // the tail has a single N tile: one bias vector for every task
    for (int i = ctid; i < p.ch.n2; i += 128 * kConsumers) s_bias2[i] = (i < p.ch.bias2_len) ? __ldg(p.ch.bias2 + i) : 0.f;
  }
  const bool fixed_n = kLean || (gridDim.x % p.n_tiles) == 0;
  if (fixed_n) {
    const int n0f = kLean ? 0 : (blockIdx.x % p.n_tiles) * p.block_n;
    for (int i = ctid; i < p.block_n; i += 128 * kConsumers) s_bias[i] = (n0f + i < p.bias_len) ? __ldg(p.bias + n0f + i) : 0.f;
  }
  consumer_sync();
  if (p.b_resident || p.band) mbar_wait(&b_full[0], 0);
  if constexpr (kChain) mbar_wait(&w2_full, 0);

  int ka = 0, kb = 0, store_idx = 0;
  uint32_t xph = 0;
  for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
    const int m_first = kLean ? task : (task / p.n_tiles) * p.pair;
    const int cnt = p.s2 ? 2 : (kLean ? 1 : min(p.pair, p.m_tiles - m_first));
    const int n0 = kLean ? 0 : (task % p.n_tiles) * p.block_n;
    if (!fixed_n) {
      consumer_sync();
      for (int i = ctid; i < p.block_n; i += 128 * kConsumers) s_bias[i] = (n0 + i < p.bias_len) ? __ldg(p.bias + n0 + i) : 0.f;
    }
    const int tmode = mode == 1 && cnt == 1 ? 0 : mode;   // the odd last pair holds one tile
    for (int c = 0; c < p.chunks; ++c) {
      const int sa0 = ka % p.a_slots, sa1 = (ka + 1) % p.a_slots;
      mbar_wait(&a_full[sa0], (ka / p.a_slots) & 1);
      if (cnt == 2) mbar_wait(&a_full[sa1], ((ka + 1) / p.a_slots) & 1);
      const uint32_t a_lo0 = smem_lo16(a_buf + static_cast<size_t>(sa0) * p.a_stride) + a_wg16;
      const uint32_t a_lo1 = smem_lo16(a_buf + static_cast<size_t>(sa1) * p.a_stride) + a_wg16;
      const bool first_chunk = c == 0;
      wgmma_fence();
      if (!kLean && p.band) {
        // Super-pixel stem (engine.stem_superpixel, pack 4, 16 channels per pixel, one 64-channel chunk): the expanded
        // weight matrix is block-banded -- a group of 4 output pixels reads, per filter row, exactly the 6 input pixels
        // x 16 channels that sit in 192 CONTIGUOUS bytes of the patch, starting 96 bytes into the left neighbour
        // super-pixel.  Six K=16 steps per filter row walk that span; the weights hold only those K-slices: [ky][2
        // blocks of 64], the last 32 columns of the second block are zero padding that is never multiplied.
        const uint32_t prow16 = static_cast<uint32_t>(pitch) * row16;
        for (int ky = 0; ky < 3; ++ky) {
          for (int j = 0; j < 6; ++j) {
            const uint32_t al = a_lo0 + ky * prow16 + 6 + 2 * j;
            const uint32_t b_lo = b_res_lo0 + static_cast<uint32_t>(ky * 2 + (j >> 2)) * b_step16 + 2 * (j & 3);
            wgmma_mma<kBf16, kN>(acc, desc_lohi(al, a_hi), desc_lohi(b_lo, b_hi), ky != 0 || j != 0);
          }
        }
        wgmma_commit();
      } else {
        const int kc = c == p.chunks - 1 ? p.kk_last : kk;
        if (kLean || p.b_resident) {
          // all nine weight slabs are in shared memory
          const uint32_t b_lo_chunk = b_res_lo0 + static_cast<uint32_t>(c * 9) * b_step16;
          for (int tap = 0; tap < 9; ++tap)
            issue_tap<kBf16, kN, kPair>(tmode, tap, kc, first_chunk && tap == 0, acc, a_lo0 + tap_off16(tap), a_lo1 + tap_off16(tap),
                             a_hi, b_lo_chunk + tap * b_step16, b_hi);
          wgmma_commit();
        } else {
          // weights streamed through the ring: per tap wait for its slab, issue, and release the previous tap's slab
          // once the MMAs that read it have completed
          int prev_sb = -1;
          for (int tap = 0; tap < 9; ++tap, ++kb) {
            const int sb = kb % p.b_stages;
            mbar_wait(&b_full[sb], (kb / p.b_stages) & 1);
            issue_tap<kBf16, kN, kPair>(tmode, tap, kc, first_chunk && tap == 0, acc, a_lo0 + tap_off16(tap), a_lo1 + tap_off16(tap),
                             a_hi, b_res_lo0 + static_cast<uint32_t>(sb) * b_step16, b_hi);
            wgmma_commit();
            wgmma_wait<1>();
            if (prev_sb >= 0 && wg_leader) mbar_arrive(&b_empty[prev_sb]);
            prev_sb = sb;
          }
          wgmma_wait<0>();
          if (wg_leader) mbar_arrive(&b_empty[prev_sb]);
        }
      }
      wgmma_wait<0>();
      if (wg_leader) {
        mbar_arrive(&a_empty[sa0]);
        if (cnt == 2) mbar_arrive(&a_empty[sa1]);
      }
      ka += cnt;
    }
    fence_acc<kTileAcc>(acc);
    if (!fixed_n) consumer_sync();   // bias visible

    const int n_tiles_here = kPair && p.pair == 2 ? cnt : 1;
    int x0 = 0, y0 = 0, n_img = 0;
    for (int tsel = 0; tsel < n_tiles_here; ++tsel) {
      tile_coords(p, m_first + tsel, n_img, y0, x0);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int y = y0 + yy[rr], x = x0 + xx[rr];
        fr.ok[rr] = yy[rr] < p.tg.tile_h && y < p.H && x < p.W;
        fr.row[rr] = (static_cast<long long>(n_img) * p.H + y) * p.W + x;
      }
      if constexpr (kChain) {
        // chain tasks index the staging buffers by box (own box first, then the extra operand block; they stay put until
        // the tail GEMM has read them), so the previous task's stores must have drained the buffers first
        if (issuer) {
          tma_store_wait_read<0>();
          if (p.ch.extra_on) {   // the cv2 half of the concat for this tile's pixels: same box as the output tile
            mbar_expect_tx(&x_full, p.ch.extra_bytes);
            tma_load_tiled_4d(&tmap_x, &x_full, staging + p.ch.own_chunks * kStageBufBytes, 0, x0, y0, n_img);
          }
        }
        consumer_sync();
      }
      if (tsel == 0)
        store_tile<kBf16, kChain, kN>(p, &tmap_out, acc, s_bias, fr, n0, x0, y0, n_img, staging, store_idx, issuer, lane);
      else if constexpr (kPair)
        store_tile<kBf16, kChain, kN>(p, &tmap_out, acc + kN / 2, s_bias, fr, n0, x0, y0, n_img, staging, store_idx, issuer, lane);
    }
    if constexpr (kChain) {
      // the tile's box(es) are in shared memory and visible to the async proxy: multiply them with the tail weights
      if (p.ch.extra_on) {
        mbar_wait(&x_full, xph);
        xph ^= 1u;
      }
      const uint32_t a2_hi = desc_hi(p.ch.own_row_bytes, 8 * p.ch.own_row_bytes);
      const uint32_t x_hi = desc_hi(p.ch.extra_row_bytes, 8 * p.ch.extra_row_bytes);
      const uint32_t w2_lo0 = smem_lo16(w2_res);
      float acc2[kChain ? kN2 / 2 : 8];   // the tail's own accumulator: the tile's is dead by now
      wgmma_fence();
      for (int j = 0; j < p.ch.w2_chunks; ++j) {
        const bool own = j < p.ch.own_chunks;
        const uint32_t rb = own ? p.ch.own_row_bytes : p.ch.extra_row_bytes;
        const uint32_t a_lo = smem_lo16(staging + j * kStageBufBytes) + ((64 * g * rb) >> 4);
        for (int k = 0; k < p.ch.ksteps; ++k)
          wgmma_mma<kBf16, kChain ? kN2 : 16>(acc2, desc_lohi(a_lo + 2 * k, own ? a2_hi : x_hi),
                            desc_lohi(w2_lo0 + j * (p.ch.w2_sub_bytes >> 4) + 2 * k, desc_hi(p.ch.w2_row_bytes, 8 * p.ch.w2_row_bytes)),
                            (j | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc<kChain ? kN2 / 2 : 8>(acc2);
      // the tail's boxes reuse the staging buffers: the operand blocks are dead (both warpgroups' tail GEMMs have
      // completed), but the stores of the first output may still be reading them
      if (issuer) tma_store_wait_read<0>();
      consumer_sync();
      for (int c0 = 0; c0 < p.ch.n2; c0 += 64) {
        uint8_t* buf = staging + ((c0 / 64) & 1) * kStageBufBytes;
        epilogue_box<kBf16, kChain ? kN2 : 16>(p.ch.ep2, acc2, c0, 64, s_bias2, fr, 0, buf, lane);
        fence_proxy_async_smem();
        if (issuer) tma_store_wait_read<0>();   // box k + 1 overwrites the buffer of box k - 1
        consumer_sync();
        if (issuer) {
          if (c0 < p.ch.ep2.Cout) tma_store_4d(&tmap_out2, buf, c0, x0, y0, n_img);
          tma_store_commit();
        }
      }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

// ===================== four consumer warpgroups: 128-column pair tasks =====================
// The stride-1 layers whose weights are streamed (pair tasks) with a Cout that splits into 128-column N tiles.  A task
// is a pair of M tiles times one 128-column N tile; consumer warpgroup w multiplies rows 64 (w mod 2) .. +63 of tile
// w / 2 with m64n128k16 (64 accumulators per thread, as many as a 64-column pair), and all four read the same weight
// slab per tap.  Per FLOP the weight and patch streams are those of the 64-column pairs, the MMAs are twice as wide
// (an m64n128k16 reads 96 B of shared memory per clock against the 64-column MMA's 128 B), and the main loop keeps one
// commit group in flight across channel chunks: a patch slot is released once the group of the chunk's last tap has
// completed, not after a drain.  Every output element gets the k16 steps of the 64-column pair launch in the same
// order (chunk, tap, k), so the outputs are the same bits.  Warpgroups 2w and 2w + 1 form team w: they own tile w's
// epilogue, staging buffers and named barrier.  Only what this path needs is compiled: no chained tail, banded stem,
// stride 2, resident weights or per-task bias reload (every CTA keeps one N tile, see patch_conv_plan).
constexpr int kQuadConsumers = 4;
constexpr int kQuadThreads = 128 * (1 + kQuadConsumers);   // 640
constexpr uint32_t kQuadAllBar = 3;                          // the 512 consumer threads; teams use barriers 1 and 2
// 227 KB per CTA (the H100's opt-in maximum) less this kernel's static shared memory (barriers + bias, ptxas -v)
constexpr size_t kQuadStaticSmem = (2 * kMaxA + 2 * kMaxB) * 8 + kMaxBlockN * 4;
constexpr size_t kQuadSmemBudget = 227 * 1024 - kQuadStaticSmem;

template <bool kBf16>
__global__ void __launch_bounds__(kQuadThreads, 1)
conv3x3_patch_quad_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                          const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap,
                          const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap, const PatchParams p) {
  constexpr int kN = 128;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[kMaxA], a_empty[kMaxA];
  __shared__ __align__(8) uint64_t b_full[kMaxB], b_empty[kMaxB];
  __shared__ __align__(16) float s_bias[kN];

  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* a_buf = base;                                                        // [a_slots][a_stride]
  uint8_t* b_buf = a_buf + static_cast<size_t>(p.a_slots) * p.a_stride;          // ring [b_stages][b_sub_bytes]
  uint8_t* staging = b_buf + static_cast<size_t>(p.b_stages) * p.b_sub_bytes;   // [2 teams][store_bufs][stage_buf_bytes]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int taps_total = 9 * p.chunks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < p.a_slots; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 2);                // the two warpgroups of the team whose tile the patch is
    }
    for (int s = 0; s < kMaxB; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], kQuadConsumers);   // every consumer warpgroup reads every slab
    }
    mbar_fence_init();
  }
  __syncthreads();
  // programmatic dependent launch as in conv3x3_patch_kernel: the weight producer does not wait for the previous grid
  if (warp != 2) asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // 640 threads start with 96 registers each; 128 x 24 + 512 x 112 = 60 416 <= 640 x 96.  The producers lower their
  // budget and return before the consumers raise theirs.
  if (warp < 4) asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");

  if (warp == 0) {
    // ===================== patch (A) producer: the two tiles of a pair per channel chunk =====================
    int ka = 0;
    for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
      const int m_first = (task / p.n_tiles) * 2;
      const int cnt = min(2, p.m_tiles - m_first);
      for (int c = 0; c < p.chunks; ++c) {
        for (int j = 0; j < cnt; ++j, ++ka) {
          int n_img, y0, x0;
          tile_coords(p, m_first + j, n_img, y0, x0);
          const int s = ka % p.a_slots;
          mbar_wait(&a_empty[s], ((ka / p.a_slots) & 1) ^ 1);
          if (YB_ELECT()) {
            mbar_expect_tx(&a_full[s], p.a_bytes);
            tma_load_tiled_4d(&tmap_a, &a_full[s], a_buf + static_cast<size_t>(s) * p.a_stride, c * p.block_k, x0 - 1,
                              y0 - 1, n_img);
          }
        }
      }
    }
    return;
  }
  if (warp == 2) {
    // ===================== weight (B) producer: one 128-column slab per (chunk, tap) =====================
    const uint32_t b_bytes = p.block_n * p.block_k * 2;
    int kb = 0;
    for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
      const int n0 = (task % p.n_tiles) * p.block_n;
      for (int i = 0; i < taps_total; ++i, ++kb) {
        const int s = kb % p.b_stages;
        mbar_wait(&b_empty[s], ((kb / p.b_stages) & 1) ^ 1);
        if (YB_ELECT()) {
          mbar_expect_tx(&b_full[s], b_bytes);
          tma_load_2d(&tmap_b, &b_full[s], b_buf + static_cast<size_t>(s) * p.b_sub_bytes,
                      ((i % 9) * p.chunks + i / 9) * p.block_k, n0);
        }
      }
    }
    return;
  }
  if (warp < 4) return;
  asm volatile("setmaxnreg.inc.sync.aligned.u32 112;\n" ::: "memory");

  // ===================== consumers =====================
  const int cw = (warp >> 2) - 1;   // consumer warpgroup 0..3
  const int team = cw >> 1, half = cw & 1;
  const int wq = warp & 3;
  const int ctid = threadIdx.x - 128;
  const bool issuer = (ctid & 255) == 0;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  FragRows fr;
  fr.loc[0] = half * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  float acc[kN / 2];

  // grid % n_tiles == 0 (host): task % n_tiles, the N tile, is the same for every task of this CTA
  const int n0 = (blockIdx.x % p.n_tiles) * p.block_n;
  for (int i = ctid; i < kN; i += 128 * kQuadConsumers) s_bias[i] = (n0 + i < p.bias_len) ? __ldg(p.bias + n0 + i) : 0.f;
  named_bar_sync(kQuadAllBar, 128 * kQuadConsumers);

  int ka = 0, kb = 0, store_idx = 0;
  for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
    const int m_first = (task / p.n_tiles) * 2;
    const int cnt = min(2, p.m_tiles - m_first);
    // Team 1 has no tile in the odd last pair.  It still issues its MMAs, on whatever its next patch slot holds, without
    // waiting for or releasing that slot, and discards the result: a branch around the MMAs would make ptxas serialise
    // every wgmma of the kernel (C7520).  It reads and releases every weight slab like the other warpgroups.
    const bool active = team < cnt;
    int prev_sb = -1, prev_sa = -1;   // slab / patch slot read by the commit group still in flight
    // descriptor constants, derived per task rather than held through the epilogue (registers are short)
    const uint32_t row_bytes = p.block_k * 2;
    const uint32_t sbo = p.tg.sbo_rows * row_bytes;
    const uint32_t a_wg16 = (8 * sbo * half) >> 4;   // this warpgroup's 64 rows: 8 groups of 8 further into every view
    const uint32_t row16 = row_bytes >> 4;
    const uint32_t a_hi = desc_hi(row_bytes, sbo);
    const uint32_t b_hi = desc_hi(row_bytes, 8 * row_bytes);
    const uint32_t b_lo0 = smem_lo16(b_buf);
    const uint32_t b_step16 = p.b_sub_bytes >> 4;
    for (int c = 0; c < p.chunks; ++c) {
      const int sa = (ka + team) % p.a_slots;
      if (active) mbar_wait(&a_full[sa], ((ka + team) / p.a_slots) & 1);
      const uint32_t a_lo = smem_lo16(a_buf + static_cast<size_t>(sa) * p.a_stride) + a_wg16;
      const int kc = c == p.chunks - 1 ? p.kk_last : (p.block_k >> 4);
      wgmma_fence();
      for (int tap = 0; tap < 9; ++tap, ++kb) {
        const int sb = kb % p.b_stages;
        mbar_wait(&b_full[sb], (kb / p.b_stages) & 1);
        const int dy = tap / 3, dx = tap - dy * 3;
        const uint32_t a_tap = a_lo + static_cast<uint32_t>(dy * p.tg.pitch + dx) * row16;
        const uint32_t b_lo = b_lo0 + static_cast<uint32_t>(sb) * b_step16;
        for (int k = 0; k < kc; ++k)
          wgmma_mma<kBf16, kN>(acc, desc_lohi(a_tap + 2 * k, a_hi), desc_lohi(b_lo + 2 * k, b_hi),
                               !(c == 0 && tap == 0 && k == 0));
        wgmma_commit();
        wgmma_wait<1>();   // the previous group (previous tap, possibly of the previous chunk) has completed
        if (wg_leader) {
          if (prev_sb >= 0) mbar_arrive(&b_empty[prev_sb]);
          if (prev_sa >= 0) mbar_arrive(&a_empty[prev_sa]);
        }
        prev_sb = sb;
        prev_sa = -1;
      }
      prev_sa = active ? sa : -1;   // released once the group of this chunk's last tap has completed
      ka += cnt;
    }
    wgmma_wait<0>();
    if (wg_leader) {
      mbar_arrive(&b_empty[prev_sb]);
      if (prev_sa >= 0) mbar_arrive(&a_empty[prev_sa]);
    }
    fence_acc<kN / 2>(acc);

    // an inactive team runs the epilogue too (a branch around it would put the next task's MMAs on a divergent path,
    // C7520), with no rows in range and no store
    int n_img, y0, x0;
    tile_coords(p, m_first + team, n_img, y0, x0);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {   // the row's place in the tile, recomputed here: registers are short
      const int grp = fr.loc[rr] >> 3;
      const int yy = grp / p.tg.gpr, xx = (grp - yy * p.tg.gpr) * 8 + (fr.loc[rr] & 7);
      const int y = y0 + yy, x = x0 + xx;
      fr.ok[rr] = active && yy < p.tg.tile_h && y < p.H && x < p.W;
      fr.row[rr] = (static_cast<long long>(n_img) * p.H + y) * p.W + x;
    }
    uint8_t* team_staging = staging + static_cast<size_t>(team) * p.store_bufs * p.stage_buf_bytes;
    // the team's tile in two boxes of 64 columns through its two staging buffers (as store_tile: before the barrier
    // the issuer waits until the previous store has read its buffer, which the next box overwrites).  Unrolled, so
    // that the first box's 32 accumulators are dead while the second box is written.
#pragma unroll
    for (int c0 = 0; c0 < kN; c0 += 64, ++store_idx) {
      uint8_t* buf = team_staging + (store_idx & 1) * p.stage_buf_bytes;
      epilogue_box<kBf16, kN>(p.ep, acc, c0, 64, s_bias, fr, n0, buf, lane);
      fence_proxy_async_smem();
      if (issuer) tma_store_wait_read<0>();
      named_bar_sync(1 + team, 256);   // the team's barrier
      if (issuer) {
        if (active && n0 + c0 < p.ep.Cout) tma_store_4d(&tmap_out, buf, n0 + c0, x0, y0, n_img);
        tma_store_commit();
      }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

// ===================== two consumer teams: single-tile tasks over one resident weight copy =====================
// The one-CTA launches with resident weights that cannot take two CTAs per SM (two copies of the weights do not fit):
// the banded stem (kN = 128, kN2 = 0) and the chained 3x3 launches after a 64-column N tile (kN = 64, tail of kN2
// columns).  The quad instance's layout: one producer warpgroup and four consumer warpgroups; warpgroups 2t and 2t + 1
// form team t, which owns a whole 128-row tile exactly as the two consumer warpgroups of conv3x3_patch_kernel do.
// The teams walk the CTA's task list alternately (team t takes positions t, t + 2, ...), so one team's epilogue, tail
// GEMM and store waits overlap the other team's MMAs.  Shared: the resident weights (3x3 or stem band), the tail
// weights, the bias vectors and the patch producer; per team: a named barrier (1 + t), two 16 KB staging buffers, the
// extra operand's mbarrier and a TMA-store issuer, whose bulk async-groups are its own.  The patch ring is shared and
// filled in task order; a slot is released by the team that read it.  Its slot count is a multiple of 2 x chunks
// (patch_conv_plan), so every slot is only ever filled for one team: a team's parity wait on a slot then follows the
// fill it waited on last, whereas a slot whose previous fill was the other team's could still have that fill in
// flight, and the parity of the fill before it would let the wait pass.  Every output element gets the MMA sequence
// and epilogue of conv3x3_patch_kernel, so the outputs are the same bits.  Only what these launches need is compiled:
// stride 1, classic tiles, one N tile with resident weights, single-tile tasks, the chained tail or the band loop.
constexpr uint32_t kTeamAllBar = 3;   // the 512 consumer threads; the teams use barriers 1 and 2
constexpr int kTeamMinTasksPerSm = 8;  // patch_conv_plan
constexpr size_t kTeamStaticSmem = (2 * kMaxA + 4) * 8 + 2 * kMaxBlockN * 4;
constexpr size_t kTeamSmemBudget = 227 * 1024 - kTeamStaticSmem;

template <bool kBf16, int kN, int kN2>
__global__ void __launch_bounds__(kQuadThreads, 1)
conv3x3_patch_team_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                          const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_w2,
                          const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_out2,
                          const PatchParams p) {
  constexpr bool kChain = kN2 != 0;
  constexpr bool kBand = !kChain;   // the stem has no tail; every chained launch here has a 64-column N tile
  // chains: the 64-column first output, plus (128-column tails) the extra operand block, as 64-channel K chunks
  constexpr int kTailChunks = kN2 == 128 ? 2 : 1;
  static_assert(kBand ? kN == 128 : kN == 64, "team instances: the stem (N = 128) or a chain after N = 64");
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[kMaxA], a_empty[kMaxA];
  __shared__ __align__(8) uint64_t b_full, w2_full;
  __shared__ __align__(8) uint64_t x_full[2];   // per team: the extra operand block has landed
  __shared__ __align__(16) float s_bias[kN];
  __shared__ __align__(16) float s_bias2[kChain ? kN2 : 4];

  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* a_buf = base;                                              // [a_slots][a_stride]
  uint8_t* b_buf = a_buf + static_cast<size_t>(p.a_slots) * p.a_stride;  // resident [9 * chunks] or the band's [6]
  uint8_t* staging = b_buf + p.b_res_bytes;                           // [2 teams][2][kStageBufBytes]
  uint8_t* w2_res = staging + 4 * kStageBufBytes;                     // chain: tail weights

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < p.a_slots; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 2);   // the two warpgroups of the team whose tile the patch is
    }
    mbar_init(&b_full, 1);
    mbar_init(&w2_full, 1);
    mbar_init(&x_full[0], 1);
    mbar_init(&x_full[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  // programmatic dependent launch as in conv3x3_patch_kernel: the weight producer does not wait for the previous grid
  if (warp != 2) asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // the quad instance's split: 128 x 24 + 512 x 112 <= 640 x 96; the producers lower their budget and return before
  // the consumers raise theirs
  if (warp < 4) asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");

  if (warp == 0) {
    // ===================== patch (A) producer: the CTA's tasks in order, whichever team runs them =====================
    int ka = 0;
    for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
      int n_img, y0, x0;
      tile_coords(p, task, n_img, y0, x0);
      for (int c = 0; c < p.chunks; ++c, ++ka) {
        const int s = ka % p.a_slots;
        mbar_wait(&a_empty[s], ((ka / p.a_slots) & 1) ^ 1);
        if (YB_ELECT()) {
          mbar_expect_tx(&a_full[s], p.a_bytes);
          tma_load_tiled_4d(&tmap_a, &a_full[s], a_buf + static_cast<size_t>(s) * p.a_stride, c * p.block_k, x0 - 1,
                            y0 - 1, n_img);
        }
      }
    }
    return;
  }
  if (warp == 2) {
    // ===================== weights, once: the 3x3 slabs or the stem band, and the tail's =====================
    if (lane == 0) {
      const uint32_t b_bytes = p.block_n * p.block_k * 2;
      if constexpr (kChain) {
        tma_prefetch_desc(&tmap_w2);
        tma_prefetch_desc(&tmap_out2);
        if (p.ch.extra_on) tma_prefetch_desc(&tmap_x);
        mbar_expect_tx(&w2_full, p.ch.w2_chunks * p.ch.n2 * p.ch.w2_row_bytes);
        for (int j = 0; j < p.ch.w2_chunks; ++j)
          tma_load_2d(&tmap_w2, &w2_full, w2_res + j * p.ch.w2_sub_bytes, j * (p.ch.w2_row_bytes >> 1), 0);
        const int taps_total = 9 * p.chunks;
        mbar_expect_tx(&b_full, taps_total * b_bytes);
        for (int i = 0; i < taps_total; ++i)   // i = chunk*9 + tap ; weight column block = tap*chunks + chunk
          tma_load_2d(&tmap_b, &b_full, b_buf + static_cast<size_t>(i) * p.b_sub_bytes,
                      ((i % 9) * p.chunks + i / 9) * p.block_k, 0);
      } else {   // banded stem weights: 3 filter rows x 2 blocks of 64 K-columns
        mbar_expect_tx(&b_full, 6 * b_bytes);
        for (int i = 0; i < 6; ++i)
          tma_load_2d(&tmap_b, &b_full, b_buf + static_cast<size_t>(i) * p.b_sub_bytes, i * p.block_k, 0);
      }
    }
    return;
  }
  if (warp < 4) return;
  asm volatile("setmaxnreg.inc.sync.aligned.u32 112;\n" ::: "memory");

  // ===================== consumers: team t, warpgroup `half` of it multiplies rows 64 half .. +63 =====================
  const int cw = (warp >> 2) - 1;
  const int team = cw >> 1, half = cw & 1;
  const int wq = warp & 3;
  const int ctid = threadIdx.x - 128;
  const bool issuer = (ctid & 255) == 0;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint32_t team_bar = 1 + team;
  FragRows fr;
  fr.loc[0] = half * 64 + wq * 16 + (lane >> 2);
  fr.loc[1] = fr.loc[0] + 8;
  uint8_t* team_staging = staging + static_cast<size_t>(team) * 2 * kStageBufBytes;
  float acc[kN / 2];

  for (int i = ctid; i < kN; i += 128 * kQuadConsumers) s_bias[i] = (i < p.bias_len) ? __ldg(p.bias + i) : 0.f;
  if constexpr (kChain) {
    for (int i = ctid; i < kN2; i += 128 * kQuadConsumers) s_bias2[i] = (i < p.ch.bias2_len) ? __ldg(p.ch.bias2 + i) : 0.f;
  }
  named_bar_sync(kTeamAllBar, 128 * kQuadConsumers);
  mbar_wait(&b_full, 0);
  if constexpr (kChain) mbar_wait(&w2_full, 0);

  uint32_t xph = 0;
  // this team's tasks: positions team, team + 2, ... of the CTA's list; ka = the position's first patch
  for (int task = blockIdx.x + team * gridDim.x, ka = team * p.chunks; task < p.num_tasks;
       task += 2 * gridDim.x, ka += 2 * p.chunks) {
    {
      // descriptor constants, derived per task rather than held through the epilogue (registers are short)
      const uint32_t row_bytes = p.block_k * 2;
      const uint32_t sbo = p.tg.sbo_rows * row_bytes;
      const uint32_t a_wg16 = (8 * sbo * half) >> 4;   // this warpgroup's 64 rows: 8 groups of 8 further into every view
      const uint32_t row16 = row_bytes >> 4;
      const uint32_t a_hi = desc_hi(row_bytes, sbo);
      const uint32_t b_hi = desc_hi(row_bytes, 8 * row_bytes);
      const uint32_t b_lo0 = smem_lo16(b_buf);
      const uint32_t b_step16 = p.b_sub_bytes >> 4;
      // The first MMA overwrites the accumulators; zeroing them first tells ptxas that the previous task's values are
      // dead, which it cannot see through the run-time accumulate flag (otherwise they stay live across the tail GEMM
      // and spill).  The band loop's flag is a compile-time constant.
      if constexpr (kChain) {
#pragma unroll
        for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
      }
      for (int c = 0; c < p.chunks; ++c) {
        const int kq = ka + c;
        const int sa = kq % p.a_slots;
        mbar_wait(&a_full[sa], (kq / p.a_slots) & 1);
        const uint32_t a_lo = smem_lo16(a_buf + static_cast<size_t>(sa) * p.a_stride) + a_wg16;
        wgmma_fence();
        if constexpr (kBand) {
          // the band MMA loop of conv3x3_patch_kernel: per filter row six K=16 steps over 192 contiguous patch bytes
          const uint32_t prow16 = static_cast<uint32_t>(p.tg.pitch) * row16;
          for (int ky = 0; ky < 3; ++ky) {
            for (int j = 0; j < 6; ++j) {
              const uint32_t al = a_lo + ky * prow16 + 6 + 2 * j;
              const uint32_t b_lo = b_lo0 + static_cast<uint32_t>(ky * 2 + (j >> 2)) * b_step16 + 2 * (j & 3);
              wgmma_mma<kBf16, kN>(acc, desc_lohi(al, a_hi), desc_lohi(b_lo, b_hi), ky != 0 || j != 0);
            }
          }
        } else {
          // whole 64-channel chunks (patch_conv_plan): four K steps per tap, a fixed count (C7520 as in the tail)
          const uint32_t b_lo_chunk = b_lo0 + static_cast<uint32_t>(c * 9) * b_step16;
          for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap - dy * 3;
            const uint32_t a_tap = a_lo + static_cast<uint32_t>(dy * p.tg.pitch + dx) * row16;
            const uint32_t b_lo = b_lo_chunk + static_cast<uint32_t>(tap) * b_step16;
#pragma unroll
            for (int k = 0; k < 4; ++k)
              wgmma_mma<kBf16, kN>(acc, desc_lohi(a_tap + 2 * k, a_hi), desc_lohi(b_lo + 2 * k, b_hi),
                                   !(c == 0 && tap == 0 && k == 0));
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (wg_leader) mbar_arrive(&a_empty[sa]);
      }
    }
    fence_acc<kN / 2>(acc);

    int n_img, y0, x0;
    tile_coords(p, task, n_img, y0, x0);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {   // the row's place in the tile (classic tiles: one 8-pixel group per tile row)
      const int y = y0 + (fr.loc[rr] >> 3), x = x0 + (fr.loc[rr] & 7);
      fr.ok[rr] = y < p.H && x < p.W;
      // the stem has no shortcut (patch_conv_plan), so its epilogue never reads the row address
      fr.row[rr] = kBand ? 0 : (static_cast<long long>(n_img) * p.H + y) * p.W + x;
    }
    if constexpr (kBand) {
      // two boxes of 64 columns through the team's two staging buffers, box b in buffer b (as store_tile, whose box
      // count per task is even here: before the barrier the issuer waits until the previous store has read its buffer,
      // which the next box overwrites)
#pragma unroll
      for (int c0 = 0; c0 < kN; c0 += 64) {
        uint8_t* buf = team_staging + (c0 / 64) * kStageBufBytes;
        epilogue_box<kBf16, kN>(p.ep, acc, c0, 64, s_bias, fr, 0, buf, lane);
        fence_proxy_async_smem();
        if (issuer) tma_store_wait_read<0>();
        named_bar_sync(team_bar, 256);
        if (issuer) {
          if (c0 < p.ep.Cout) tma_store_4d(&tmap_out, buf, c0, x0, y0, n_img);
          tma_store_commit();
        }
      }
    } else {
      // the first output in one box (staging buffer 0), the extra operand block in buffer 1; both stay put until the
      // tail GEMM has read them, so the team's previous stores must have drained the buffers first
      if (issuer) {
        tma_store_wait_read<0>();
        if (p.ch.extra_on) {   // the cv2 half of the concat for this tile's pixels: same box as the output tile
          mbar_expect_tx(&x_full[team], p.ch.extra_bytes);
          tma_load_tiled_4d(&tmap_x, &x_full[team], team_staging + p.ch.own_chunks * kStageBufBytes, 0, x0, y0, n_img);
        }
      }
      named_bar_sync(team_bar, 256);
      epilogue_box<kBf16, kN>(p.ep, acc, 0, p.store_cols, s_bias, fr, 0, team_staging, lane);
      fence_proxy_async_smem();
      named_bar_sync(team_bar, 256);
      if (issuer) {
        if (p.ch.store_first) tma_store_4d(&tmap_out, team_staging, 0, x0, y0, n_img);
        tma_store_commit();
      }
      if (p.ch.extra_on) {
        mbar_wait(&x_full[team], xph);
        xph ^= 1u;
      }
      const uint32_t a2_hi = desc_hi(p.ch.own_row_bytes, 8 * p.ch.own_row_bytes);
      const uint32_t x_hi = desc_hi(p.ch.extra_row_bytes, 8 * p.ch.extra_row_bytes);
      const uint32_t w2_lo0 = smem_lo16(w2_res);
      float acc2[kChain ? kN2 / 2 : 8];   // the tail's own accumulator: the tile's is dead by now
      wgmma_fence();
      // the chunk count and their 64 channels are fixed per instance (patch_conv_plan): with run-time loop bounds here
      // ptxas serialises the wgmmas (C7520)
#pragma unroll
      for (int j = 0; j < kTailChunks; ++j) {
        const bool own = j == 0;
        const uint32_t rb = own ? p.ch.own_row_bytes : p.ch.extra_row_bytes;
        const uint32_t a_lo = smem_lo16(team_staging + j * kStageBufBytes) + ((64 * half * rb) >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_mma<kBf16, kChain ? kN2 : 16>(acc2, desc_lohi(a_lo + 2 * k, own ? a2_hi : x_hi),
                                              desc_lohi(w2_lo0 + j * (p.ch.w2_sub_bytes >> 4) + 2 * k,
                                                        desc_hi(p.ch.w2_row_bytes, 8 * p.ch.w2_row_bytes)),
                                              (j | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc<kChain ? kN2 / 2 : 8>(acc2);
      // the tail's boxes reuse the team's staging buffers: the operand blocks are dead (both warpgroups' tail GEMMs
      // have completed), but the store of the first output may still be reading buffer 0
      if (issuer) tma_store_wait_read<0>();
      named_bar_sync(team_bar, 256);
      EpilogueParams ep2 = p.ch.ep2;
      ep2.residual = nullptr;   // never set for a tail (chain_setup); known here, the epilogue drops its row addresses
#pragma unroll
      for (int c0 = 0; c0 < (kChain ? kN2 : 16); c0 += 64) {
        uint8_t* buf = team_staging + ((c0 / 64) & 1) * kStageBufBytes;
        epilogue_box<kBf16, kChain ? kN2 : 16>(ep2, acc2, c0, 64, s_bias2, fr, 0, buf, lane);
        fence_proxy_async_smem();
        if (issuer) tma_store_wait_read<0>();   // box k + 1 overwrites the buffer of box k - 1
        named_bar_sync(team_bar, 256);
        if (issuer) {
          if (c0 < p.ch.ep2.Cout) tma_store_4d(&tmap_out2, buf, c0, x0, y0, n_img);
          tma_store_commit();
        }
      }
    }
  }
  if (issuer) tma_store_wait_all<0>();
}

}  // namespace

using PatchKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                               const CUtensorMap, const PatchParams);

// One kernel per (dtype, N tile, chained tail N, CTAs per SM): the MMA width and the accumulator size are compile-time
// constants of every instance.  patch_conv_configure admits exactly these shapes.
// Pair tasks with a 128-column N tile run on four consumer warpgroups (the plan caps the two-group pairs at 64 columns).
static bool quad_plan(const PatchParams& kp) { return kp.pair == 2 && !kp.s2 && kp.block_n == 128; }

// Two consumer teams run the banded stem and the chains after a 64-column N tile (patch_conv_plan sets kp.teams).
static bool four_groups(const PatchParams& kp) { return quad_plan(kp) || kp.teams; }

template <bool kBf16>
PatchKernelFn select_patch_kernel_t(const PatchParams& kp) {
  if (quad_plan(kp)) return conv3x3_patch_quad_kernel<kBf16>;
  if (kp.teams) {
    if (kp.band) return conv3x3_patch_team_kernel<kBf16, 128, 0>;
    return kp.ch.n2 == 64 ? conv3x3_patch_team_kernel<kBf16, 64, 64> : conv3x3_patch_team_kernel<kBf16, 64, 128>;
  }
  if (kp.ctas == 2) {
    // two CTAs per SM: the instances whose consumers fit in 104 registers without spilling (N = 32 / 64, N = 32 with a
    // 64-column tail; DESIGN.md section 3)
    if (kp.ch.on) return kp.block_n == 32 && kp.ch.n2 == 64 ? conv3x3_patch_kernel<kBf16, 32, 64, 2> : nullptr;
    switch (kp.block_n) {
      case 32: return conv3x3_patch_kernel<kBf16, 32, 0, 2>;
      case 64: return conv3x3_patch_kernel<kBf16, 64, 0, 2>;
      default: return nullptr;
    }
  }
  if (kp.ch.on) {
    if (kp.block_n == 32) return kp.ch.n2 == 64 ? conv3x3_patch_kernel<kBf16, 32, 64, 1> : conv3x3_patch_kernel<kBf16, 32, 128, 1>;
    return kp.ch.n2 == 64 ? conv3x3_patch_kernel<kBf16, 64, 64, 1> : conv3x3_patch_kernel<kBf16, 64, 128, 1>;
  }
  switch (kp.block_n) {
    case 32: return conv3x3_patch_kernel<kBf16, 32, 0, 1>;
    case 64: return conv3x3_patch_kernel<kBf16, 64, 0, 1>;
    default: return conv3x3_patch_kernel<kBf16, 128, 0, 1>;
  }
}
PatchKernelFn select_patch_kernel(const PatchParams& kp) {
  return kp.ep.is_bf16 ? select_patch_kernel_t<true>(kp) : select_patch_kernel_t<false>(kp);
}

namespace {
// Fraction of the accumulator rows that are real output pixels, per tiling.
double classic_eff(int H, int W) {
  const int ty = (H + 15) / 16, tx = (W + 7) / 8;
  return static_cast<double>(H) * W / (static_cast<double>(ty) * tx * 128);
}
double wrap_eff(int H, int W) {
  if (W > 22 || W < 9) return 0.0;
  return static_cast<double>(H) * W / (static_cast<double>((H + 4) / 5) * 128);
}
TileGeom pick_geom(int H, int W, bool allow_wrap, bool s2) {
  TileGeom g;
  if (s2) {   // H, W: output extent; the patch is one column-parity plane of the input
    g.tile_h = 16; g.tile_w = 8; g.x_step = 8; g.pitch = 9; g.patch_h = 33; g.gpr = 1; g.sbo_rows = 18;
    g.alloc_rows = 33 * 9;
  } else if (allow_wrap && wrap_eff(H, W) > classic_eff(H, W)) {
    g.tile_h = 5; g.tile_w = 24; g.x_step = 24; g.pitch = 24; g.patch_h = 7; g.gpr = 3; g.sbo_rows = 8;
    g.alloc_rows = 8 * 24;    // rows 120..127 of the tap view (2,2) reach pixel-row 7*24 + 9
  } else {
    g.tile_h = 16; g.tile_w = 8; g.x_step = 8; g.pitch = 10; g.patch_h = 18; g.gpr = 1; g.sbo_rows = 10;
    g.alloc_rows = 18 * 10;
  }
  return g;
}
}  // namespace

// Eligibility: 3x3 / stride 1 / pad 1 and a feature map that one of the two tilings covers with little waste.
bool patch_conv_eligible(const yb_op_desc& d) {
  if (d.kind != YB_OP_CONV || d.ksize != 3 || d.pad != 1) return false;
  if (d.reserved & YB_CONV_FORCE_IM2COL) return false;   // caller asked for the generic im2col kernel
  if (d.stride == 2)   // two column-parity planes: even width, and an output map that 16 x 8 tiles cover well.
    // With two channel chunks (four 38 KB planes per tile) or a split N tile the planes leave little room for the
    // pipeline, so those stay on the im2col kernel unless the caller forces the variant (YB_CONV_FORCE_PLANES).
    return (d.reserved & YB_CONV_BAND_STEM) == 0 && d.W % 2 == 0 && d.H % 2 == 0 && classic_eff(d.Ho, d.Wo) >= 0.7 &&
           ((d.Cin <= 64 && d.Cout <= 128) || (d.reserved & YB_CONV_FORCE_PLANES));
  if (d.stride != 1) return false;
  const bool band = (d.reserved & YB_CONV_BAND_STEM) != 0;
  const double eff = band ? classic_eff(d.H, d.W) : (classic_eff(d.H, d.W) > wrap_eff(d.H, d.W) ? classic_eff(d.H, d.W) : wrap_eff(d.H, d.W));
  return eff >= 0.7;
}

static int patch_conv_plan(const yb_op_desc& d, int ctas, PatchParams& kp, dim3& grid, size_t& smem_bytes);

// Pure host logic: tiling, shared-memory layout and launch shape (no driver calls).  Two CTAs per SM when the shape has
// a two-CTA instance, its plan fits half of the SM's shared memory with resident weights and there are tasks for both
// (YB_CONV_ONE_CTA keeps one CTA per SM: tests compare the two launches bit for bit).
static int patch_conv_configure(const yb_op_desc& d, PatchParams& kp, dim3& grid, size_t& smem_bytes) {
  if (!(d.reserved & YB_CONV_ONE_CTA) && patch_conv_plan(d, 2, kp, grid, smem_bytes) == YB_OK) return YB_OK;
  return patch_conv_plan(d, 1, kp, grid, smem_bytes);
}

// The plan for `ctas` CTAs per SM.  With ctas = 2 it gets half of the SM's shared memory, less the per-CTA reservation
// and the kernel's static shared memory, and fails unless the weights stay resident in one N tile, the tasks are single
// tiles, the shape has a two-CTA instance and there are at least 2 x SMs tasks.
static int patch_conv_plan(const yb_op_desc& d, int ctas, PatchParams& kp, dim3& grid, size_t& smem_bytes) {
  const size_t budget = ctas == 2 ? smem_per_sm() / 2 - kSmemReservedPerCta - kStaticSmem : kSmemBudget;
  kp = PatchParams();
  kp.ctas = ctas;
  kp.N = d.N;
  kp.s2 = d.stride == 2 ? 1 : 0;
  kp.H = d.Ho;     // the kernel tiles the OUTPUT map (equal to the input extent at stride 1)
  kp.W = d.Wo;
  // the weights are the banded super-pixel stem matrix [Cout_pad][3 rows][2 x 64] (engine.stem_band)
  kp.band = (d.reserved & YB_CONV_BAND_STEM) ? 1 : 0;
  kp.tg = pick_geom(kp.H, kp.W, !kp.band, kp.s2 != 0);
  const TileGeom& tg = kp.tg;
  kp.tiles_x = (kp.W + tg.x_step - 1) / tg.x_step;
  kp.tiles_y = (kp.H + tg.tile_h - 1) / tg.tile_h;
  kp.m_tiles = d.N * kp.tiles_x * kp.tiles_y;
  const int sms = num_sms();
  // N tile: 32..128 columns (wider accumulators than 64 registers per thread would not leave room for the patch
  // kernel's addressing next to the in-flight wgmma; narrower ones cost more than they save)
  int n_tiles = (d.Cout + kMaxBlockN - 1) / kMaxBlockN;
  int block_n = mma_n((d.Cout + n_tiles - 1) / n_tiles);
  if (block_n < 32) block_n = 32;
  if (block_n > kMaxBlockN) block_n = kMaxBlockN;
  n_tiles = (d.Cout + block_n - 1) / block_n;
  kp.block_k = (d.Cin_pad % 64 == 0) ? 64 : ((d.Cin_pad % 32 == 0) ? 32 : 16);
  kp.chunks = d.Cin_pad / kp.block_k;
  kp.kk_last = (d.Cin - (kp.chunks - 1) * kp.block_k + 15) / 16;
  if (kp.kk_last < 1) kp.kk_last = 1;
  if (kp.kk_last > (kp.block_k >> 4)) kp.kk_last = kp.block_k >> 4;
  kp.a_bytes = tg.patch_h * tg.pitch * kp.block_k * 2;
  kp.a_stride = (static_cast<uint32_t>(tg.alloc_rows * kp.block_k * 2) + 1023u) & ~1023u;
  kp.store_bufs = kp.s2 ? 1 : 2;   // the two 38 KB planes of the stride-2 variant take the second staging buffer's room
  kp.bias_len = d.Cout_pad;
  const size_t staging = static_cast<size_t>(kp.store_bufs) * kStageBufBytes;
  // chained tail: its resident weights come out of the same budget (chain_setup validates the rest below, once the
  // first convolution's tiling is known; the byte count only depends on the descriptor)
  size_t chain_bytes = 0;
  if (d.chain != nullptr) {
    const int kc = d.chain->own_C >= 64 ? 64 : d.chain->own_C;
    const int chunks2 = kc > 0 ? d.chain->K_pad / kc : 0;
    chain_bytes = static_cast<size_t>(chunks2) * ((static_cast<size_t>(mma_n(d.chain->Cout_pad)) * kc * 2 + 1023) & ~static_cast<size_t>(1023));
    YB_REQUIRE(chain_bytes + staging + 1024 + 64 * 1024 < budget, "patch conv: chained tail weights (%zu bytes) do not fit", chain_bytes);
  }
  const size_t avail = budget - staging - 1024 - chain_bytes;
  uint32_t b_sub = (static_cast<uint32_t>(block_n * kp.block_k * 2) + 1023u) & ~1023u;
  size_t b_total = static_cast<size_t>(kp.band ? 6 : 9 * kp.chunks) * b_sub;
  kp.b_resident = (n_tiles == 1 && b_total + 2 * kp.a_stride <= avail) ? 1 : 0;
  kp.stage_buf_bytes = kStageBufBytes;
  // N-split with resident weights: when the whole filter bank does not fit in shared memory but half (a quarter) of it
  // does, every CTA keeps ONE N tile for all its tasks (grid % n_tiles == 0 makes task % n_tiles constant per CTA) and
  // loads that slice once; the patch is then fetched by n_tiles CTAs, but nothing is streamed per task any more.  Only
  // taken when three patch slots still fit next to the slice (see below) -- which rules out the zoo's 128-channel
  // layers (144 KB slice + 3 x 23 KB patches + staging > 222 KB): those keep the pair-of-tiles weight stream.
  int forced_store_cols = 0;
  size_t staging_ns = staging;
  if (!kp.b_resident && !kp.band && !kp.s2 && d.chain == nullptr && !(d.reserved & YB_CONV_NO_NSPLIT)) {
    for (int ns = 2; ns <= 4 && !kp.b_resident; ns *= 2) {
      if (d.Cout % (16 * ns) || sms % ns) continue;
      const int bn = d.Cout / ns;
      if (bn < 64) break;                      // narrower MMAs / more patch re-reads than the weight stream costs
      if (mma_n(bn) != bn || bn > kMaxBlockN) continue;   // the slice must be an N tile of this kernel
      const uint32_t bs = (static_cast<uint32_t>(bn * kp.block_k * 2) + 1023u) & ~1023u;
      const size_t bt = static_cast<size_t>(9 * kp.chunks) * bs;
      const int opt_cols[3] = {64, 64, 32}, opt_bufs[3] = {2, 1, 1};
      for (int o = 0; o < 3; ++o) {
        if (bn % opt_cols[o]) continue;
        const size_t buf_bytes = static_cast<size_t>(128) * opt_cols[o] * 2;
        const size_t stg = static_cast<size_t>(opt_bufs[o]) * buf_bytes;
        // at least three patch slots: with two, a task that needs both (two channel chunks) cannot prefetch the next
        // task's patch and every task pays the L2 latency
        if (bt + 3 * kp.a_stride + stg + 1024 > budget) continue;
        n_tiles = ns;
        block_n = bn;
        b_sub = bs;
        b_total = bt;
        kp.b_resident = 1;
        kp.store_bufs = opt_bufs[o];
        kp.stage_buf_bytes = static_cast<int>(buf_bytes);
        forced_store_cols = opt_cols[o];
        staging_ns = stg;
        break;
      }
    }
  }
  const size_t avail_ns = budget - staging_ns - 1024 - chain_bytes;
  // Weights that do not fit in shared memory are streamed from L2 for every task; two M tiles per weight pass halve
  // that stream (the bound of the deep layers: 128 -> 128 at 40 x 40 re-reads 295 KB per 128 output pixels).  Pair
  // tasks hold the accumulators of two tiles in registers, so their N tile is at most 64 columns (stride-2 tasks with
  // streamed weights: 128).
  kp.pair = (!kp.b_resident && !kp.band && !kp.s2 && kp.m_tiles >= 2) ? 2 : 1;
  // Pairs whose Cout splits into 128-column N tiles run on four consumer warpgroups instead (conv3x3_patch_quad_kernel)
  // when the grid is a multiple of the N tiles (one N tile per CTA), the 128-column tasks fill the grid (T >= G) and
  // cost no extra round of it: T tasks of 128 columns run ceil(T / G) rounds of twice the work of the 2T tasks of 64
  // columns, which run ceil(2T / G) rounds, so 2 ceil(T / G) <= ceil(2T / G), i.e. T mod G = 0 or T mod G > G / 2.
  // c2 on 132 SMs: the 40² layers (240 tasks) take it, the 20² ones (128 tasks) do not.  YB_CONV_PAIR_N64 keeps the
  // 64-column pairs.
  const int quad_tiles = d.Cout / 128;
  const int quad_tasks = ((kp.m_tiles + 1) / 2) * quad_tiles;
  const int grid_q = quad_tasks < sms ? quad_tasks : sms;
  const bool quad = ctas == 1 && kp.pair == 2 && d.chain == nullptr && d.Cout % 128 == 0 &&
                    !(d.reserved & YB_CONV_PAIR_N64) && grid_q % quad_tiles == 0 && quad_tasks >= sms &&
                    2 * ((quad_tasks + sms - 1) / sms) <= (2 * quad_tasks + sms - 1) / sms;
  const int n_cap = kp.pair == 2 && !quad ? 64 : 128;
  if ((kp.pair == 2 || (kp.s2 && !kp.b_resident)) && block_n > n_cap) {
    n_tiles = (d.Cout + n_cap - 1) / n_cap;
    block_n = mma_n((d.Cout + n_tiles - 1) / n_tiles);
    n_tiles = (d.Cout + block_n - 1) / block_n;
    b_sub = (static_cast<uint32_t>(block_n * kp.block_k * 2) + 1023u) & ~1023u;
    b_total = static_cast<size_t>(9 * kp.chunks) * b_sub;
  }
  YB_REQUIRE(mma_n(block_n) == block_n && block_n <= kMaxBlockN, "patch conv: N tile %d is not a wgmma N", block_n);
  kp.block_n = block_n;
  kp.n_tiles = n_tiles;
  kp.b_sub_bytes = b_sub;
  kp.store_cols = forced_store_cols ? forced_store_cols : ((block_n % 64 == 0) ? 64 : ((block_n % 32 == 0) ? 32 : 16));
  kp.num_tasks = ((kp.m_tiles + kp.pair - 1) / kp.pair) * n_tiles;
  if (kp.band && !(d.Cin_pad == 64 && n_tiles == 1 && kp.store_cols == 64 && d.act < YB_ACT_HARDSWISH &&
                   d.residual == nullptr)) {
    set_error("patch conv: banded stem weights need Cin_pad 64, one N tile with 64-column store boxes, SiLU/linear epilogue");
    return YB_ERR_INVALID;
  }
  if (kp.band && !kp.b_resident) {
    set_error("patch conv: banded stem weights do not fit in shared memory (block_n=%d)", block_n);
    return YB_ERR_INVALID;
  }
  kp.ch.on = 0;
  if (d.chain != nullptr) {
    YB_REQUIRE(kp.b_resident && kp.pair == 1 && !kp.s2 && !kp.band,
               "patch conv: a chained tail needs resident weights and single-tile stride-1 tasks (block_n=%d resident=%d pair=%d)",
               block_n, kp.b_resident, kp.pair);
    YB_REQUIRE(kp.store_cols == block_n && (block_n == 64 || block_n == 32),
               "patch conv: a chained tail needs the first output in one 32- or 64-column box, got block_n=%d", block_n);
    const char* why = chain_setup(d, block_n, n_tiles, kp.store_cols, /*allow_extra=*/true, &kp.ch);
    YB_REQUIRE(why == nullptr, "patch conv: chained tail not supported here: %s", why);
    YB_REQUIRE(kp.ch.n2 == 64 || kp.ch.n2 == 128, "patch conv: the tail must have 33-128 output columns, got %d", kp.ch.n2);
    YB_REQUIRE(static_cast<size_t>(kp.ch.w2_chunks) * kp.ch.w2_sub_bytes == chain_bytes, "patch conv: tail weight layout mismatch");
    // the extra block arrives as the output tile's box: tile_w x tile_h pixel-rows (120 for the wrap tiling; the rows
    // beyond are never stored)
    kp.ch.extra_bytes = static_cast<uint32_t>(tg.tile_w * tg.tile_h) * static_cast<uint32_t>(kp.ch.extra_row_bytes);
  }
  kp.b_res_bytes = kp.b_resident ? static_cast<uint32_t>(b_total) : 0u;
  kp.ep.is_bf16 = d.dtype == YB_BF16;
  if (ctas == 2 && !(kp.b_resident && n_tiles == 1 && kp.pair == 1 && !kp.band && kp.num_tasks >= 2 * sms &&
                     select_patch_kernel(kp) != nullptr))
    return YB_ERR_INVALID;
  // Two consumer teams (conv3x3_patch_team_kernel) for the one-CTA launches with resident weights in one N tile and
  // single-tile classic tasks that are the 128-column banded stem, or a chain after a 64-column N tile over whole
  // 64-channel chunks whose tail reads one 64-channel chunk (64-column tails) or two (128-column tails: the first
  // output and the extra operand) -- the shapes the team instances compile -- when each team's two staging buffers
  // and one patch slot per channel chunk fit next to the weights in 227 KB and the launch has at least
  // kTeamMinTasksPerSm tasks per SM.
  // The threshold keeps the smaller launches (the fingerprint plans' stems and chains, about 800 tasks) on two
  // warpgroups; DESIGN.md section 3 has the measured sweep.  YB_CONV_NO_TEAMS keeps two consumer warpgroups, and so
  // does YB_CONV_PAIR_N64, which names the two-warpgroup launch of every four-warpgroup one.
  const bool team_chain = kp.ch.on && block_n == 64 && kp.block_k == 64 && kp.kk_last == 4 && kp.ch.ksteps == 4 &&
                          kp.ch.w2_chunks == (kp.ch.n2 == 128 ? 2 : 1);
  const size_t team_fixed = b_total + 2 * staging + chain_bytes + 1024;
  kp.teams = ctas == 1 && !(d.reserved & (YB_CONV_NO_TEAMS | YB_CONV_PAIR_N64)) && kp.b_resident && n_tiles == 1 &&
             kp.pair == 1 && !kp.s2 && tg.x_step == 8 && ((kp.band && block_n == 128) || team_chain) &&
             kp.num_tasks >= kTeamMinTasksPerSm * sms && 2 * kp.chunks <= kMaxA &&
             team_fixed + 2 * static_cast<size_t>(kp.chunks) * kp.a_stride <= kTeamSmemBudget;
  if (kp.teams) {
    // a multiple of 2 x chunks patch slots: each slot then serves one team only (see conv3x3_patch_team_kernel)
    const int a_st = static_cast<int>((kTeamSmemBudget - team_fixed) / kp.a_stride);
    kp.a_slots = (a_st > kMaxA ? kMaxA : a_st) / (2 * kp.chunks) * (2 * kp.chunks);
    kp.b_stages = 1;
    staging_ns = 2 * staging;
  } else if (kp.b_resident) {
    int a_st = static_cast<int>((avail_ns - b_total) / kp.a_stride);
    kp.a_slots = a_st > kMaxA ? kMaxA : a_st;
    kp.b_stages = 1;
  } else if (quad) {
    // four patch slots (this chunk's two tiles and the next chunk's) and two 16 KB staging buffers per team; the weight
    // ring gets the rest of the 227 KB: 231 680 - 1024 - 4 x 23 552 - 65 536 = 70 912 B with classic tiles, 66 816 B
    // with wrap tiles (24 KB patches), i.e. four 16 KB slabs (a slab feeds 16 MMAs, about 0.55 us at the dense rate)
    kp.a_slots = 4;
    staging_ns = 2 * staging;
    const size_t used = 1024 + static_cast<size_t>(kp.a_slots) * kp.a_stride + staging_ns;
    const int b_st = used < kQuadSmemBudget ? static_cast<int>((kQuadSmemBudget - used) / kp.b_sub_bytes) : 0;
    kp.b_stages = b_st > kMaxB ? kMaxB : b_st;
    YB_REQUIRE(kp.b_stages >= 2, "patch conv: not enough shared memory for the weight ring of four consumer warpgroups");
  } else {
    // patch slots: a pair task holds two at a time, a third (fourth) lets the next chunk's patches stream in meanwhile;
    // the weight ring gets the rest (every slab is consumed within ~0.1-0.3 us, the ring covers the L2 latency)
    kp.a_slots = (kp.pair == 2 || kp.s2) ? 3 : 2;
    size_t rem = avail - static_cast<size_t>(kp.a_slots) * kp.a_stride;
    if (rem >= static_cast<size_t>(kp.a_stride) + 6 * kp.b_sub_bytes) {
      kp.a_slots += 1;
      rem -= kp.a_stride;
    }
    int b_st = static_cast<int>(rem / kp.b_sub_bytes);
    kp.b_stages = b_st > kMaxB ? kMaxB : b_st;
    if (kp.b_stages < 2) {
      set_error("patch conv: not enough shared memory for the weight ring (block_n=%d)", block_n);
      return YB_ERR_INVALID;
    }
  }
  YB_REQUIRE(kp.a_slots >= 2, "patch conv: fewer than two patch slots fit in shared memory (block_n=%d)", block_n);
  YB_REQUIRE(!kp.teams || kp.a_slots % (2 * kp.chunks) == 0, "patch conv: %d patch slots do not divide between two teams",
             kp.a_slots);
  kp.ep.Cout = d.Cout;
  kp.ep.act = d.act;
  kp.ep.residual = d.residual;
  kp.ep.res_cstride = d.res_cstride;
  kp.bias = d.bias;
  const int max_grid = ctas * sms;
  grid = dim3(kp.num_tasks < max_grid ? kp.num_tasks : max_grid, 1, 1);
  YB_REQUIRE(!(kp.b_resident && n_tiles > 1) || grid.x % n_tiles == 0, "patch conv: N-split grid %u not a multiple of %d", grid.x, n_tiles);
  const size_t b_region = kp.b_resident ? kp.b_res_bytes : static_cast<size_t>(kp.b_stages) * kp.b_sub_bytes;
  const size_t smem = static_cast<size_t>(kp.a_slots) * kp.a_stride + b_region + staging_ns + chain_bytes + 1024;
  const size_t cap = quad ? kQuadSmemBudget : (kp.teams ? kTeamSmemBudget : budget);
  YB_REQUIRE(smem <= cap, "patch conv: %zu bytes of shared memory needed, %zu available", smem, cap);
  smem_bytes = smem;
  return YB_OK;
}

int patch_conv_config(const yb_op_desc& d, yb_conv_info* info) {
  PatchParams kp;
  dim3 grid;
  size_t smem = 0;
  int rc = conv_validate(d);
  if (rc == YB_OK) rc = patch_conv_configure(d, kp, grid, smem);
  if (rc == YB_OK && info) {   // yb_conv_config: see include/yolort_b200.h
    info->kernel = YB_CONV_KERNEL_PATCH;
    info->block_n = kp.block_n;
    info->n_tiles = kp.n_tiles;
    info->weights_resident = kp.b_resident;
    info->tiles_per_pass = kp.pair;
    info->slots = kp.a_slots;
    info->ring = kp.b_resident ? 0 : kp.b_stages;
    info->store_cols = kp.store_cols;
    info->store_bufs = kp.store_bufs;
    info->groups = four_groups(kp) ? kQuadConsumers : kConsumers;
    info->resident_ctas = kp.ctas;
    info->chained = kp.ch.on;
    info->smem_bytes = static_cast<int>(smem);
    info->grid = static_cast<int>(grid.x);
    info->tiling = kp.s2 ? YB_CONV_TILING_STRIDE2 : (kp.tg.x_step == 24 ? YB_CONV_TILING_WRAP : YB_CONV_TILING_CLASSIC);
    info->m_tiles = kp.m_tiles;
    info->work_items = kp.num_tasks;
    info->tail_n = kp.ch.n2;
  }
  return rc;
}

struct PatchConvOp final : ConvOp {
  CUtensorMap tmap_a, tmap_b, tmap_out, tmap_w2, tmap_x, tmap_out2;
  PatchParams kp;
  PatchKernelFn fn = nullptr;
  dim3 grid;
  size_t smem_bytes;
  int launch(cudaStream_t stream) const override {
    YB_CHECK_CUDA(launch_pdl(fn, grid, dim3(four_groups(kp) ? kQuadThreads : kThreads), smem_bytes, stream, tmap_a, tmap_b,
                             tmap_out, tmap_w2, tmap_x, tmap_out2, kp));
    return YB_OK;
  }
};

int patch_conv_create(const yb_op_desc& d, ConvOp** out) {
  PatchConvOp* op = new PatchConvOp();
  PatchParams& kp = op->kp;
  int rc = conv_validate(d);
  if (rc == YB_OK) rc = patch_conv_configure(d, kp, op->grid, op->smem_bytes);
  const TileGeom& tg = kp.tg;
  const CUtensorMapDataType dt = kp.ep.is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const uint32_t bk = kp.block_k;
  if (rc == YB_OK && kp.s2) {
    // [C, column parity, W/2, H, N] over the NHWC input: a box with parity extent 1 is one plane's patch
    const cuuint64_t dims[5] = {static_cast<cuuint64_t>(d.Cin), 2, static_cast<cuuint64_t>(d.W / 2),
                                static_cast<cuuint64_t>(d.H), static_cast<cuuint64_t>(d.N)};
    const cuuint32_t box[5] = {bk, 1, static_cast<cuuint32_t>(tg.pitch), static_cast<cuuint32_t>(tg.patch_h), 1};
    rc = tmap_tiled(&op->tmap_a, "patch conv stride-2 input planes", dt, d.in, 5, dims, d.in_cstride, box,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  } else if (rc == YB_OK) {
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(d.W), static_cast<cuuint64_t>(d.H),
                                static_cast<cuuint64_t>(d.N)};
    const cuuint32_t box[4] = {bk, static_cast<cuuint32_t>(tg.pitch), static_cast<cuuint32_t>(tg.patch_h), 1};
    rc = tmap_tiled(&op->tmap_a, "patch conv input patch", dt, d.in, 4, dims, d.in_cstride, box,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  }
  const int ktot = kp.band ? 6 * 64 : 9 * d.Cin_pad;
  if (rc == YB_OK)
    rc = tmap_matrix(&op->tmap_b, "patch conv weights", dt, d.weight, ktot, d.Cout_pad, ktot, bk, kp.block_n,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  // NHWC views of the output extent, in boxes of the output tile's tile_w x tile_h pixels
  const cuuint64_t out_px[3] = {static_cast<cuuint64_t>(d.Wo), static_cast<cuuint64_t>(d.Ho), static_cast<cuuint64_t>(d.N)};
  auto out_view = [&](CUtensorMap* map, const char* what, const void* base, int C, int cstride, uint32_t box_c,
                      CUtensorMapL2promotion l2) {
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), out_px[0], out_px[1], out_px[2]};
    const cuuint32_t box[4] = {box_c, static_cast<cuuint32_t>(tg.tile_w), static_cast<cuuint32_t>(tg.tile_h), 1};
    return tmap_tiled(map, what, dt, base, 4, dims, cstride, box, l2);
  };
  if (rc == YB_OK)
    rc = out_view(&op->tmap_out, "patch conv output", d.out, d.Cout, d.out_cstride, kp.store_cols,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE);
  op->tmap_w2 = op->tmap_b;      // placeholders when nothing is chained (never dereferenced)
  op->tmap_x = op->tmap_a;
  op->tmap_out2 = op->tmap_out;
  if (rc == YB_OK && kp.ch.on) {
    const yb_conv_chain& c = *d.chain;
    const uint32_t kc = kp.ch.w2_row_bytes / 2;
    rc = tmap_matrix(&op->tmap_w2, "patch conv chained tail weights", dt, c.weight, c.K_pad, c.Cout_pad, c.K_pad, kc,
                     kp.ch.n2, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc == YB_OK && kp.ch.extra_on)   // the tile's pixels of the extra operand: the output tile's box
      rc = out_view(&op->tmap_x, "patch conv chained tail extra operand", c.extra, c.extra_C, c.extra_cstride, kc,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    if (rc == YB_OK)
      rc = out_view(&op->tmap_out2, "patch conv chained tail output", c.out, c.Cout, c.out_cstride, 64,
                    CU_TENSOR_MAP_L2_PROMOTION_NONE);
  }
  if (rc == YB_OK) {
    op->fn = select_patch_kernel(kp);
    const bool quad = four_groups(kp);
    rc = set_smem_attributes(reinterpret_cast<const void*>(op->fn),
                             quad_plan(kp) ? kQuadSmemBudget : (kp.teams ? kTeamSmemBudget : kSmemBudget), kp.ctas,
                             op->smem_bytes, quad ? kQuadThreads : kThreads, "patch conv");
    if (rc == YB_OK && quad) {   // the 640-thread CTA with up to 227 KB of shared memory must fit on an SM
      int per_sm = 0;
      const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, op->fn, kQuadThreads, op->smem_bytes);
      if (e != cudaSuccess) {
        set_error("patch conv: cudaOccupancyMaxActiveBlocksPerMultiprocessor failed: %s", cudaGetErrorString(e));
        rc = YB_ERR_CUDA;
      } else if (per_sm < 1) {
        set_error("patch conv: the four-warpgroup CTA (%d threads, %zu bytes of shared memory) does not fit on an SM",
                  kQuadThreads, op->smem_bytes);
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
