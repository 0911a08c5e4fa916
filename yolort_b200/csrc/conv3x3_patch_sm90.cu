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
// Roles (one persistent CTA per SM, 384 threads): warp 0 = patch (A) producer, warp 2 = weight (B) producer (unless
// the weights are resident in shared memory), warpgroups 1-2 = consumers: each multiplies 64 of the tile's 128
// accumulator rows with wgmma (fp32 accumulators in registers) and runs the epilogue on its fragment.
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
//   mode 0: one tile; 1: two tiles sharing the weight slab (second accumulator at acc + kN / 2, kN <= 64);
//   2: stride 2, one accumulator, the tap picks its column-parity plane (a0 = even plane, a1 = odd plane).
template <bool kBf16, int kN>
__device__ __forceinline__ void issue_tap(int mode, int tap, int kc, bool first, float* acc, uint32_t a0, uint32_t a1,
                                          uint32_t a_hi, uint32_t b_lo, uint32_t b_hi) {
  for (int k = 0; k < kc; ++k) {
    const bool accum = !(first && k == 0);
    const uint64_t db = desc_lohi(b_lo + 2 * k, b_hi);
    if (mode == 2) {
      wgmma_mma<kBf16, kN>(acc, desc_lohi(((tap % 3) == 1 ? a0 : a1) + 2 * k, a_hi), db, accum);
    } else {
      wgmma_mma<kBf16, kN>(acc, desc_lohi(a0 + 2 * k, a_hi), db, accum);
      if constexpr (kN <= 64) {
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

// kN: the wgmma N of the tile (= block_n; pair tasks, kN <= 64, hold two tiles' accumulators).  kN2 != 0: a pointwise
// tail of kN2 columns is chained onto every tile (conv_chain.cuh):
// tmap_w2 = its weights, tmap_x = its optional second operand block (C3: the cv2 half of the concat, fetched per tile
// with the output tile's box), tmap_out2 = its output.
template <bool kBf16, int kN, int kN2>
__global__ void __launch_bounds__(kThreads, 1)
conv3x3_patch_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_w2,
                     const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_out2,
                     const PatchParams p) {
  constexpr bool kChain = kN2 != 0;
  constexpr int kTileAcc = kN <= 64 ? kN : kN / 2;   // accumulator registers per thread: two tiles when kN <= 64
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
  if (warp < 4)
    regs_producer();
  else
    regs_consumer();

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
  const bool fixed_n = (gridDim.x % p.n_tiles) == 0;
  if (fixed_n) {
    const int n0f = (blockIdx.x % p.n_tiles) * p.block_n;
    for (int i = ctid; i < p.block_n; i += 128 * kConsumers) s_bias[i] = (n0f + i < p.bias_len) ? __ldg(p.bias + n0f + i) : 0.f;
  }
  consumer_sync();
  if (p.b_resident || p.band) mbar_wait(&b_full[0], 0);
  if constexpr (kChain) mbar_wait(&w2_full, 0);

  int ka = 0, kb = 0, store_idx = 0;
  uint32_t xph = 0;
  for (int task = blockIdx.x; task < p.num_tasks; task += gridDim.x) {
    const int m_first = (task / p.n_tiles) * p.pair;
    const int cnt = p.s2 ? 2 : min(p.pair, p.m_tiles - m_first);
    const int n0 = (task % p.n_tiles) * p.block_n;
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
      if (p.band) {
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
        if (p.b_resident) {
          // all nine weight slabs are in shared memory
          const uint32_t b_lo_chunk = b_res_lo0 + static_cast<uint32_t>(c * 9) * b_step16;
          for (int tap = 0; tap < 9; ++tap)
            issue_tap<kBf16, kN>(tmode, tap, kc, first_chunk && tap == 0, acc, a_lo0 + tap_off16(tap), a_lo1 + tap_off16(tap),
                             a_hi, b_lo_chunk + tap * b_step16, b_hi);
          wgmma_commit();
        } else {
          // weights streamed through the ring: per tap wait for its slab, issue, and release the previous tap's slab
          // once the MMAs that read it have completed
          int prev_sb = -1;
          for (int tap = 0; tap < 9; ++tap, ++kb) {
            const int sb = kb % p.b_stages;
            mbar_wait(&b_full[sb], (kb / p.b_stages) & 1);
            issue_tap<kBf16, kN>(tmode, tap, kc, first_chunk && tap == 0, acc, a_lo0 + tap_off16(tap), a_lo1 + tap_off16(tap),
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

    const int n_tiles_here = p.pair == 2 ? cnt : 1;
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
      else if constexpr (kN <= 64)
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

}  // namespace

using PatchKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                               const CUtensorMap, const PatchParams);

// One kernel per (dtype, N tile, chained tail N): the MMA width and the accumulator size are compile-time constants of
// every instance.  patch_conv_configure admits exactly these shapes.
template <bool kBf16>
PatchKernelFn select_patch_kernel_t(const PatchParams& kp) {
  if (kp.ch.on) {
    if (kp.block_n == 32) return kp.ch.n2 == 64 ? conv3x3_patch_kernel<kBf16, 32, 64> : conv3x3_patch_kernel<kBf16, 32, 128>;
    return kp.ch.n2 == 64 ? conv3x3_patch_kernel<kBf16, 64, 64> : conv3x3_patch_kernel<kBf16, 64, 128>;
  }
  switch (kp.block_n) {
    case 32: return conv3x3_patch_kernel<kBf16, 32, 0>;
    case 64: return conv3x3_patch_kernel<kBf16, 64, 0>;
    default: return conv3x3_patch_kernel<kBf16, 128, 0>;
  }
}
PatchKernelFn select_patch_kernel(const PatchParams& kp) {
  return kp.ep.is_bf16 ? select_patch_kernel_t<true>(kp) : select_patch_kernel_t<false>(kp);
}

struct PatchConvOp {
  CUtensorMap tmap_a, tmap_b, tmap_out, tmap_w2, tmap_x, tmap_out2;
  PatchParams kp;
  PatchKernelFn fn = nullptr;
  dim3 grid;
  size_t smem_bytes;
};

namespace {
// wgmma N of an output tile: the next power of two >= 16 (weight rows past Cout_pad are zero-filled by the TMA unit, the
// store clips columns past Cout)
int mma_n(int n) {
  int c = 16;
  while (c < n) c <<= 1;
  return c;
}
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
  if (d.reserved & 1) return false;   // caller asked for the generic im2col kernel
  if (d.stride == 2)   // two column-parity planes: even width, and an output map that 16 x 8 tiles cover well.
    // With two channel chunks (four 38 KB planes per tile) or a split N tile the planes leave little room for the
    // pipeline, so those stay on the im2col kernel unless the caller forces the variant (bit 2).
    return (d.reserved & 2) == 0 && d.W % 2 == 0 && d.H % 2 == 0 && classic_eff(d.Ho, d.Wo) >= 0.7 &&
           ((d.Cin <= 64 && d.Cout <= 128) || (d.reserved & 4));
  if (d.stride != 1) return false;
  const bool band = (d.reserved & 2) != 0;
  const double eff = band ? classic_eff(d.H, d.W) : (classic_eff(d.H, d.W) > wrap_eff(d.H, d.W) ? classic_eff(d.H, d.W) : wrap_eff(d.H, d.W));
  return eff >= 0.7;
}

// Pure host logic: tiling, shared-memory layout and launch shape (no driver calls).
static int patch_conv_configure(const yb_op_desc& d, PatchParams& kp, dim3& grid, size_t& smem_bytes) {
  kp = PatchParams();
  kp.N = d.N;
  kp.s2 = d.stride == 2 ? 1 : 0;
  kp.H = d.Ho;     // the kernel tiles the OUTPUT map (equal to the input extent at stride 1)
  kp.W = d.Wo;
  // reserved bit 1: the weights are the banded super-pixel stem matrix [Cout_pad][3 rows][2 x 64] (engine.stem_band)
  kp.band = (d.reserved & 2) ? 1 : 0;
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
    YB_REQUIRE(chain_bytes + staging + 1024 + 64 * 1024 < kSmemBudget, "patch conv: chained tail weights (%zu bytes) do not fit", chain_bytes);
  }
  const size_t avail = kSmemBudget - staging - 1024 - chain_bytes;
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
  if (!kp.b_resident && !kp.band && !kp.s2 && d.chain == nullptr && !(d.reserved & 8)) {
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
        if (bt + 3 * kp.a_stride + stg + 1024 > kSmemBudget) continue;
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
  const size_t avail_ns = kSmemBudget - staging_ns - 1024 - chain_bytes;
  // Weights that do not fit in shared memory are streamed from L2 for every task; two M tiles per weight pass halve
  // that stream (the bound of the deep layers: 128 -> 128 at 40 x 40 re-reads 295 KB per 128 output pixels).  Pair
  // tasks hold the accumulators of two tiles in registers, so their N tile is at most 64 columns (stride-2 tasks with
  // streamed weights: 128).
  kp.pair = (!kp.b_resident && !kp.band && !kp.s2 && kp.m_tiles >= 2) ? 2 : 1;
  const int n_cap = kp.pair == 2 ? 64 : 128;
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
  if (kp.b_resident) {
    int a_st = static_cast<int>((avail_ns - b_total) / kp.a_stride);
    kp.a_slots = a_st > kMaxA ? kMaxA : a_st;
    kp.b_stages = 1;
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
  kp.ep.Cout = d.Cout;
  kp.ep.act = d.act;
  kp.ep.is_bf16 = d.dtype == YB_BF16;
  kp.ep.residual = d.residual;
  kp.ep.res_cstride = d.res_cstride;
  kp.bias = d.bias;
  grid = dim3(kp.num_tasks < sms ? kp.num_tasks : sms, 1, 1);
  YB_REQUIRE(!(kp.b_resident && n_tiles > 1) || grid.x % n_tiles == 0, "patch conv: N-split grid %u not a multiple of %d", grid.x, n_tiles);
  const size_t b_region = kp.b_resident ? kp.b_res_bytes : static_cast<size_t>(kp.b_stages) * kp.b_sub_bytes;
  const size_t smem = static_cast<size_t>(kp.a_slots) * kp.a_stride + b_region + staging_ns + chain_bytes + 1024;
  YB_REQUIRE(smem <= kSmemBudget, "patch conv: %zu bytes of shared memory needed, %zu available", smem, kSmemBudget);
  smem_bytes = smem;
  return YB_OK;
}

int patch_conv_configure_check(const yb_op_desc& d, int* info) {
  PatchParams kp;
  dim3 grid;
  size_t smem = 0;
  const int rc = patch_conv_configure(d, kp, grid, smem);
  if (rc == YB_OK && info) {   // yb_conv_config: see include/yolort_b200.h
    info[0] = 1;
    info[1] = kp.block_n;
    info[2] = kp.n_tiles;
    info[3] = kp.b_resident;
    info[4] = kp.pair;
    info[5] = kp.a_slots;
    info[6] = kp.b_resident ? 0 : kp.b_stages;
    info[7] = kp.store_cols;
    info[8] = kp.store_bufs;
    info[9] = static_cast<int>(smem);
    info[10] = static_cast<int>(grid.x);
    info[11] = kp.ch.on;
  }
  return rc;
}

int patch_conv_create(const yb_op_desc& d, EncodeTiledFn encode_tiled, PatchConvOp** out) {
  PatchConvOp* op = new PatchConvOp();
  PatchParams& kp = op->kp;
  int rc = patch_conv_configure(d, kp, op->grid, op->smem_bytes);
  if (rc != YB_OK) {
    delete op;
    return rc;
  }
  const TileGeom& tg = kp.tg;
  const int block_n = kp.block_n;

  const CUtensorMapDataType dt = kp.ep.is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const int rb = kp.block_k * 2;
  const CUtensorMapSwizzle sw = rb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (rb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult cr;
  if (kp.s2) {
    // [C, column parity, W/2, H, N] over the NHWC input: a box with parity extent 1 is one plane's patch
    const cuuint64_t cs = static_cast<cuuint64_t>(d.in_cstride) * 2;
    cuuint64_t dims[5] = {static_cast<cuuint64_t>(d.Cin), 2, static_cast<cuuint64_t>(d.W / 2), static_cast<cuuint64_t>(d.H),
                          static_cast<cuuint64_t>(d.N)};
    cuuint64_t strides[4] = {cs, 2 * cs, cs * d.W, cs * d.W * d.H};
    cuuint32_t box[5] = {static_cast<cuuint32_t>(kp.block_k), 1, static_cast<cuuint32_t>(tg.pitch), static_cast<cuuint32_t>(tg.patch_h), 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    cr = encode_tiled(&op->tmap_a, dt, 5, const_cast<void*>(d.in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("patch conv: cuTensorMapEncodeTiled (stride-2 input planes) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  } else {
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(d.W), static_cast<cuuint64_t>(d.H),
                          static_cast<cuuint64_t>(d.N)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(d.in_cstride) * 2, static_cast<cuuint64_t>(d.in_cstride) * 2 * d.W,
                             static_cast<cuuint64_t>(d.in_cstride) * 2 * d.W * d.H};
    cuuint32_t box[4] = {static_cast<cuuint32_t>(kp.block_k), static_cast<cuuint32_t>(tg.pitch), static_cast<cuuint32_t>(tg.patch_h), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    cr = encode_tiled(&op->tmap_a, dt, 4, const_cast<void*>(d.in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("patch conv: cuTensorMapEncodeTiled (input patch) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  {
    const int ktot = kp.band ? 6 * 64 : 9 * d.Cin_pad;
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(ktot), static_cast<cuuint64_t>(d.Cout_pad)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ktot) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(kp.block_k), static_cast<cuuint32_t>(block_n)};
    cuuint32_t estr[2] = {1, 1};
    cr = encode_tiled(&op->tmap_b, dt, 2, const_cast<void*>(d.weight), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("patch conv: cuTensorMapEncodeTiled (weights) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  {
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.Cout), static_cast<cuuint64_t>(d.Wo), static_cast<cuuint64_t>(d.Ho),
                          static_cast<cuuint64_t>(d.N)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(d.out_cstride) * 2, static_cast<cuuint64_t>(d.out_cstride) * 2 * d.Wo,
                             static_cast<cuuint64_t>(d.out_cstride) * 2 * d.Wo * d.Ho};
    cuuint32_t box[4] = {static_cast<cuuint32_t>(kp.store_cols), static_cast<cuuint32_t>(tg.tile_w), static_cast<cuuint32_t>(tg.tile_h), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    const int srb = kp.store_cols * 2;
    cr = encode_tiled(&op->tmap_out, dt, 4, d.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      srb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (srb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B),
                      CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("patch conv: cuTensorMapEncodeTiled (output) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  op->tmap_w2 = op->tmap_b;      // placeholders when nothing is chained (never dereferenced)
  op->tmap_x = op->tmap_a;
  op->tmap_out2 = op->tmap_out;
  if (kp.ch.on) {
    const yb_conv_chain& c = *d.chain;
    const int kc = kp.ch.w2_row_bytes / 2;
    const CUtensorMapSwizzle swk = kc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (kc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    cuuint64_t wdims[2] = {static_cast<cuuint64_t>(c.K_pad), static_cast<cuuint64_t>(c.Cout_pad)};
    cuuint64_t wstrides[1] = {static_cast<cuuint64_t>(c.K_pad) * 2};
    cuuint32_t wbox[2] = {static_cast<cuuint32_t>(kc), static_cast<cuuint32_t>(kp.ch.n2)};
    cuuint32_t estr2[2] = {1, 1};
    cr = encode_tiled(&op->tmap_w2, dt, 2, const_cast<void*>(c.weight), wdims, wstrides, wbox, estr2, CU_TENSOR_MAP_INTERLEAVE_NONE, swk,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    cuuint32_t estr4[4] = {1, 1, 1, 1};
    if (cr == CUDA_SUCCESS && kp.ch.extra_on) {   // the tile's pixels of the extra operand: the output tile's box
      cuuint64_t dims[4] = {static_cast<cuuint64_t>(c.extra_C), static_cast<cuuint64_t>(d.Wo), static_cast<cuuint64_t>(d.Ho),
                            static_cast<cuuint64_t>(d.N)};
      cuuint64_t strides[3] = {static_cast<cuuint64_t>(c.extra_cstride) * 2, static_cast<cuuint64_t>(c.extra_cstride) * 2 * d.Wo,
                               static_cast<cuuint64_t>(c.extra_cstride) * 2 * d.Wo * d.Ho};
      cuuint32_t box[4] = {static_cast<cuuint32_t>(kc), static_cast<cuuint32_t>(tg.tile_w), static_cast<cuuint32_t>(tg.tile_h), 1};
      cr = encode_tiled(&op->tmap_x, dt, 4, const_cast<void*>(c.extra), dims, strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE, swk,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (cr == CUDA_SUCCESS) {
      cuuint64_t dims[4] = {static_cast<cuuint64_t>(c.Cout), static_cast<cuuint64_t>(d.Wo), static_cast<cuuint64_t>(d.Ho),
                            static_cast<cuuint64_t>(d.N)};
      cuuint64_t strides[3] = {static_cast<cuuint64_t>(c.out_cstride) * 2, static_cast<cuuint64_t>(c.out_cstride) * 2 * d.Wo,
                               static_cast<cuuint64_t>(c.out_cstride) * 2 * d.Wo * d.Ho};
      cuuint32_t box[4] = {64, static_cast<cuuint32_t>(tg.tile_w), static_cast<cuuint32_t>(tg.tile_h), 1};
      cr = encode_tiled(&op->tmap_out2, dt, 4, c.out, dims, strides, box, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (cr != CUDA_SUCCESS) {
      set_error("patch conv: cuTensorMapEncodeTiled (chained tail) failed with CUresult %d", static_cast<int>(cr));
      delete op;
      return YB_ERR_CUDA;
    }
  }
  op->fn = select_patch_kernel(kp);
  cudaError_t e = cudaFuncSetAttribute(op->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBudget));
  if (e != cudaSuccess) {
    set_error("patch conv: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    delete op;
    return YB_ERR_CUDA;
  }
  *out = op;
  return YB_OK;
}

int patch_conv_launch(const PatchConvOp* op, cudaStream_t stream) {
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
  YB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, op->fn, op->tmap_a, op->tmap_b, op->tmap_out, op->tmap_w2, op->tmap_x, op->tmap_out2, op->kp));
  return YB_OK;
}

void patch_conv_destroy(PatchConvOp* op) { delete op; }

}  // namespace yb
