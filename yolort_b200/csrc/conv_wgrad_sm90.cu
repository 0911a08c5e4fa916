// Weight and bias gradient of 1x1 convolutions (the backward of the detection head's nn.Conv2d layers,
// yolort/models/box_head.py:35-37,68-82):
//
//   dW[co, ci] = sum_p dY[p, co] * X[p, ci]        db[co] = sum_p dY[p, co]
//
// p runs over the N*H*W pixels; dY and X are NHWC rows [P][stride].  The reduction dimension (pixels) is contiguous in
// neither operand, so both wgmma operands are MN-major (the transpose bits of wgmma.mma_async for 16-bit types): the
// dY tile is A (M = output channel), the X tile is B (N = input channel), and both come in by TMA straight from the row
// layouts, 64 channels x 64 pixels per box in the 128-byte swizzle.  In that layout a box is eight 1024-byte groups of
// eight pixel rows; a K = 16 step is two groups.
//
// The output is tiny (at most a few hundred x 1280) and K is huge (204,800 pixels for yolov5s level 0 at batch 32), so
// the pixels are split into slices.  One work item = (problem, 128-row output tile, up to 256-column input tile, pixel
// slice); all problems of a call (the levels of a head) form one grouped item list.
//   wgrad_partial_kernel: persistent, one CTA per SM, static round-robin over the items, 384 threads:
//     warpgroup 0 (producer): warp 0 issues the TMA loads of each 64-pixel stage into a 4-deep mbarrier ring;
//     warpgroups 1-2 (consumers): 64 output rows each, one m64n64k16 per 64-column block of the input tile, plus an
//                m64n8k16 against a resident tile of ones that yields the column sums of dY (db) on the items of the
//                first input tile.  The fp32 accumulators go to the item's partial tile in the workspace.
//   wgrad_reduce_kernel: one thread per output element sums its partials over the slices in slice order (fp32) and
//                rounds once to the output dtype.
// No float atomics: a repeated call on the same device gives the same bits.
#include "common.cuh"
#include "conv_sm90.h"

namespace yb {

namespace {

constexpr int kRows = 128;              // output rows (dY channels) per tile: two consumer warpgroups x 64
constexpr int kPx = 64;                 // pixels per pipeline stage (the K extent of one stage)
constexpr int kMaxBlocks = 4;           // 64-column input blocks per tile (up to 256 input channels)
constexpr int kBoxBytes = 64 * kPx * 2;  // one TMA box: 64 channels x 64 pixels of 16-bit values
constexpr int kStageBytes = (2 + kMaxBlocks) * kBoxBytes;
constexpr int kStages = 4;
constexpr int kOnesBytes = 2048;
constexpr size_t kSmemBytes = static_cast<size_t>(kStages) * kStageBytes + kOnesBytes + 1024;   // + alignment slack
constexpr int kThreads = 384;
constexpr int kMinSlice = 512;          // pixels: a partial tile (<= 128 KB) is written per item, keep it a minor cost

struct WgradProblemDev {
  int P, Cout, Cin;
  int co_tiles, ci_tiles, slices, slice_len;
  int n_blocks;        // 64-column blocks of Cin
  int tile_w;          // columns of one partial tile (min(n_blocks, 4) * 64)
  int item_begin;      // first work item of this problem in the grouped list
  int has_db;
  int out_begin;       // first element of this problem in the reduction's flat index space
  long long ws_off;    // floats: this problem's first partial tile in the workspace
  int item_floats;     // floats per work item: kRows x tile_w partials + kRows column sums
  void* dw;
  void* db;
};

struct WgradParams {
  CUtensorMap dy[YB_WGRAD_MAX_PROBLEMS];
  CUtensorMap x[YB_WGRAD_MAX_PROBLEMS];
  WgradProblemDev pr[YB_WGRAD_MAX_PROBLEMS];
  int n, total_items, out_total, out_dtype;
  float* ws;
};

struct Item {
  int q, local, co0, ci0, nb, px0, chunks;
};

__device__ __forceinline__ Item decode_item(const WgradParams& p, int item) {
  Item it;
  int q = 0;
  while (q + 1 < p.n && item >= p.pr[q + 1].item_begin) ++q;
  const WgradProblemDev& pr = p.pr[q];
  it.q = q;
  it.local = item - pr.item_begin;
  const int cit = it.local % pr.ci_tiles;
  const int t = it.local / pr.ci_tiles;
  const int cot = t % pr.co_tiles;
  const int s = t / pr.co_tiles;
  it.co0 = cot * kRows;
  it.ci0 = cit * 64 * kMaxBlocks;
  it.nb = min(kMaxBlocks, pr.n_blocks - cit * kMaxBlocks);
  it.px0 = s * pr.slice_len;
  const int px1 = min(it.px0 + pr.slice_len, pr.P);
  it.chunks = (px1 - it.px0 + kPx - 1) / kPx;
  return it;
}

// Descriptor of an MN-major operand in the 128-byte swizzle: 64 contiguous channels per 128-byte row, one row per
// pixel, eight-row groups 1024 bytes apart.  Every operand here is exactly one 64-wide swizzle atom in M / N, so only
// the K-group stride is read; it goes in both offset fields.
__device__ __forceinline__ uint64_t mn_desc(const void* smem) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_u32(smem) & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1024 >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= 1ull << 62;
  return d;
}
// The tile of ones (no swizzle): whatever element the MMA reads is 1.
__device__ __forceinline__ uint64_t ones_desc(const void* smem) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_u32(smem) & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(128 >> 4) << 16;
  d |= static_cast<uint64_t>(128 >> 4) << 32;
  return d;
}

// D[64 x 64] (+)= A[64 x 16] * B[16 x 64], both operands MN-major (transpose bits set).
template <bool kBf16>
__device__ __forceinline__ void wgmma_t_n64(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (!kBf16) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d));
  } else {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d));
  }
}
// D[64 x 8] (+)= A[64 x 16] * B[16 x 8], A MN-major: the column sums of A when B is all ones.
template <bool kBf16>
__device__ __forceinline__ void wgmma_t_n8(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (!kBf16) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(da), "l"(db), "r"(scale_d));
  } else {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(da), "l"(db), "r"(scale_d));
  }
}

template <bool kBf16>
__global__ void __launch_bounds__(kThreads, 1) wgrad_partial_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages];
  __shared__ __align__(8) uint64_t empty_bar[kStages];
  uint8_t* tiles = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* ones = tiles + kStages * kStageBytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  {
    const uint32_t one = kBf16 ? 0x3F803F80u : 0x3C003C00u;   // two 16-bit ones
    for (int i = threadIdx.x; i < kOnesBytes / 4; i += kThreads) reinterpret_cast<uint32_t*>(ones)[i] = one;
  }
  fence_proxy_async_smem();   // the ones are read by the tensor cores through the async proxy
  __syncthreads();

  if (warp < 4) {
    regs_producer<1>();
    if (warp != 0) return;
    // ===================== TMA producer =====================
    int kit = 0;
    for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
      const Item it = decode_item(p, item);
      const uint32_t bytes = static_cast<uint32_t>(2 + it.nb) * kBoxBytes;
      for (int c = 0; c < it.chunks; ++c, ++kit) {
        const int s = kit % kStages;
        mbar_wait(&empty_bar[s], ((kit / kStages) & 1) ^ 1);
        if (YB_ELECT()) {
          uint8_t* dst = tiles + s * kStageBytes;
          const int px = it.px0 + c * kPx;
          mbar_expect_tx(&full_bar[s], bytes);
          tma_load_2d(&p.dy[it.q], &full_bar[s], dst, it.co0, px);
          tma_load_2d(&p.dy[it.q], &full_bar[s], dst + kBoxBytes, it.co0 + 64, px);
          for (int b = 0; b < it.nb; ++b)
            tma_load_2d(&p.x[it.q], &full_bar[s], dst + (2 + b) * kBoxBytes, it.ci0 + 64 * b, px);
        }
        __syncwarp();
      }
    }
    return;
  }

  // ===================== consumers: 64 output rows each =====================
  regs_consumer<1>();
  const int g = (warp >> 2) - 1;
  const int wq = warp & 3;
  const uint64_t d_ones = ones_desc(ones);
  float acc[kMaxBlocks * 32];
  float acc_db[4];
  int kit = 0;
  for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    const Item it = decode_item(p, item);
    const WgradProblemDev& pr = p.pr[it.q];
    const bool with_db = pr.has_db && it.ci0 == 0;
    int prev_s = -1;
    for (int c = 0; c < it.chunks; ++c, ++kit) {
      const int s = kit % kStages;
      mbar_wait(&full_bar[s], (kit / kStages) & 1);
      const uint8_t* st = tiles + s * kStageBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kPx / 16; ++k) {
        const uint32_t acc_on = (c | k) != 0;
        const uint64_t da = mn_desc(st + g * kBoxBytes + k * 2048);
#pragma unroll
        for (int b = 0; b < kMaxBlocks; ++b)
          if (b < it.nb) wgmma_t_n64<kBf16>(acc + 32 * b, da, mn_desc(st + (2 + b) * kBoxBytes + k * 2048), acc_on);
        if (with_db) wgmma_t_n8<kBf16>(acc_db, da, d_ones, acc_on);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_s >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
    }
    wgmma_wait<0>();
    fence_acc<kMaxBlocks * 32>(acc);
    fence_acc<4>(acc_db);
    if (prev_s >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_s]);

    // partial tile of this item: [kRows][tile_w] fp32, then the kRows column sums
    float* part = p.ws + pr.ws_off + static_cast<long long>(it.local) * pr.item_floats;
    const int r0 = g * 64 + wq * 16 + (lane >> 2);
    const int q2 = 2 * (lane & 3);
#pragma unroll
    for (int b = 0; b < kMaxBlocks; ++b) {
      if (b < it.nb) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = 64 * b + 8 * j + q2;
          const float* a = acc + 32 * b + 4 * j;
          *reinterpret_cast<float2*>(part + static_cast<long long>(r0) * pr.tile_w + col) = make_float2(a[0], a[1]);
          *reinterpret_cast<float2*>(part + static_cast<long long>(r0 + 8) * pr.tile_w + col) = make_float2(a[2], a[3]);
        }
      }
    }
    if (with_db && (lane & 3) == 0) {
      part[kRows * pr.tile_w + r0] = acc_db[0];
      part[kRows * pr.tile_w + r0 + 8] = acc_db[2];
    }
  }
}

__device__ __forceinline__ void store_out(void* base, long long i, float v, int dtype) {
  if (dtype == YB_F32) reinterpret_cast<float*>(base)[i] = v;
  else if (dtype == YB_F16) reinterpret_cast<__half*>(base)[i] = __float2half_rn(v);
  else reinterpret_cast<__nv_bfloat16*>(base)[i] = __float2bfloat16_rn(v);
}

// One thread per output element: the sum of its partials over the slices, in slice order.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const __grid_constant__ WgradParams p) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < p.out_total; e += gridDim.x * blockDim.x) {
    int q = 0;
    while (q + 1 < p.n && e >= p.pr[q + 1].out_begin) ++q;
    const WgradProblemDev& pr = p.pr[q];
    const int local = e - pr.out_begin;
    const int n_w = pr.Cout * pr.Cin;
    int co, col, cit;
    bool bias;
    if (local < n_w) {
      co = local / pr.Cin;
      const int ci = local - co * pr.Cin;
      cit = ci / (64 * kMaxBlocks);
      col = ci - cit * 64 * kMaxBlocks;
      bias = false;
    } else {
      co = local - n_w;
      cit = 0;
      col = 0;
      bias = true;
    }
    const int cot = co / kRows, r = co - cot * kRows;
    const float* src = p.ws + pr.ws_off + static_cast<long long>(cot * pr.ci_tiles + cit) * pr.item_floats +
                       (bias ? static_cast<long long>(kRows) * pr.tile_w + r : static_cast<long long>(r) * pr.tile_w + col);
    const long long step = static_cast<long long>(pr.co_tiles) * pr.ci_tiles * pr.item_floats;
    float sum = 0.f;
    for (int s = 0; s < pr.slices; ++s) sum += __ldg(src + s * step);
    if (bias) store_out(pr.db, co, sum, p.out_dtype);
    else store_out(pr.dw, local, sum, p.out_dtype);
  }
}

int out_size(int dtype) { return dtype == YB_F32 ? 4 : 2; }

// Validation and work split (pure host logic: no driver calls).
int wgrad_configure(const yb_wgrad_problem* problems, int n, WgradParams& kp, size_t* ws_bytes) {
  YB_REQUIRE(problems != nullptr && n >= 1 && n <= YB_WGRAD_MAX_PROBLEMS,
             "conv_wgrad: needs 1 to %d problems, got %d", YB_WGRAD_MAX_PROBLEMS, problems ? n : 0);
  const int dtype = problems[0].dtype, out_dtype = problems[0].out_dtype;
  YB_REQUIRE(dtype == YB_F16 || dtype == YB_BF16, "conv_wgrad: dy / x dtype must be f16 or bf16, got %d", dtype);
  YB_REQUIRE(out_dtype == YB_F32 || out_dtype == YB_F16 || out_dtype == YB_BF16,
             "conv_wgrad: out_dtype must be f32, f16 or bf16, got %d", out_dtype);
  for (int q = 0; q < n; ++q) {
    const yb_wgrad_problem& a = problems[q];
    YB_REQUIRE(a.dtype == dtype && a.out_dtype == out_dtype, "conv_wgrad: problem %d: every problem must have the "
               "dtype and out_dtype of problem 0", q);
    YB_REQUIRE(a.P >= 1 && a.P < (1ll << 31), "conv_wgrad: problem %d: P = %lld out of range", q, static_cast<long long>(a.P));
    YB_REQUIRE(a.Cout >= 1 && a.Cin >= 1, "conv_wgrad: problem %d: Cout / Cin must be positive, got %d / %d", q, a.Cout, a.Cin);
    YB_REQUIRE(a.dy_stride % 8 == 0 && a.x_stride % 8 == 0,
               "conv_wgrad: problem %d: row strides must be multiples of 8 elements (16 bytes), got %lld / %lld", q,
               static_cast<long long>(a.dy_stride), static_cast<long long>(a.x_stride));
    YB_REQUIRE(a.Cout <= a.dy_stride, "conv_wgrad: problem %d: Cout %d exceeds the dy row stride %lld", q, a.Cout,
               static_cast<long long>(a.dy_stride));
    YB_REQUIRE(a.Cin <= a.x_stride, "conv_wgrad: problem %d: Cin %d exceeds the x row stride %lld", q, a.Cin,
               static_cast<long long>(a.x_stride));
    YB_REQUIRE(a.dy_stride < (1ll << 30) && a.x_stride < (1ll << 30), "conv_wgrad: problem %d: row stride too large", q);
    YB_REQUIRE(a.dy != nullptr && a.x != nullptr && a.dw != nullptr, "conv_wgrad: problem %d: dy, x and dw are required", q);
    YB_REQUIRE((reinterpret_cast<uintptr_t>(a.dy) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.x) & 15) == 0,
               "conv_wgrad: problem %d: dy and x must be 16-byte aligned", q);
    const uintptr_t om = static_cast<uintptr_t>(out_size(out_dtype) - 1);
    YB_REQUIRE((reinterpret_cast<uintptr_t>(a.dw) & om) == 0 && (reinterpret_cast<uintptr_t>(a.db) & om) == 0,
               "conv_wgrad: problem %d: dw / db must be aligned to their element size", q);
  }
  kp = WgradParams();
  kp.n = n;
  kp.out_dtype = out_dtype;
  const int sms = num_sms();
  // Target: about two items per CTA, sized by the bytes each one streams ((2 + input blocks) boxes per stage).
  double total = 0.0;
  for (int q = 0; q < n; ++q) {
    const yb_wgrad_problem& a = problems[q];
    const int co_tiles = (a.Cout + kRows - 1) / kRows;
    const int nbt = (a.Cin + 63) / 64;
    total += static_cast<double>(a.P) * co_tiles * (2.0 * ((nbt + kMaxBlocks - 1) / kMaxBlocks) + nbt);
  }
  const double per_item = total / (2.0 * sms);
  long long items = 0, out_total = 0, ws_floats = 0;
  for (int q = 0; q < n; ++q) {
    const yb_wgrad_problem& a = problems[q];
    WgradProblemDev& pr = kp.pr[q];
    pr.P = static_cast<int>(a.P);
    pr.Cout = a.Cout;
    pr.Cin = a.Cin;
    pr.co_tiles = (a.Cout + kRows - 1) / kRows;
    pr.n_blocks = (a.Cin + 63) / 64;
    pr.ci_tiles = (pr.n_blocks + kMaxBlocks - 1) / kMaxBlocks;
    pr.tile_w = 64 * (pr.n_blocks < kMaxBlocks ? pr.n_blocks : kMaxBlocks);
    const double per_px = (2.0 * pr.ci_tiles + pr.n_blocks) / pr.ci_tiles;   // boxes per pixel of one tile
    const long long max_slices = (a.P + kMinSlice - 1) / kMinSlice;
    long long want = static_cast<long long>(static_cast<double>(a.P) * per_px / per_item + 0.5);
    if (want < 1) want = 1;
    if (want > max_slices) want = max_slices;
    const long long len = ((a.P + want - 1) / want + kPx - 1) / kPx * kPx;
    pr.slice_len = static_cast<int>(len);
    pr.slices = static_cast<int>((a.P + len - 1) / len);
    pr.item_begin = static_cast<int>(items);
    pr.has_db = a.db != nullptr;
    pr.out_begin = static_cast<int>(out_total);
    pr.ws_off = ws_floats;
    pr.item_floats = kRows * pr.tile_w + kRows;
    pr.dw = a.dw;
    pr.db = a.db;
    const long long n_items = static_cast<long long>(pr.co_tiles) * pr.ci_tiles * pr.slices;
    items += n_items;
    ws_floats += n_items * pr.item_floats;
    out_total += static_cast<long long>(a.Cout) * a.Cin + (a.db ? a.Cout : 0);
  }
  YB_REQUIRE(items < (1ll << 31) && out_total < (1ll << 31), "conv_wgrad: problem too large");
  kp.total_items = static_cast<int>(items);
  kp.out_total = static_cast<int>(out_total);
  if (ws_bytes) *ws_bytes = static_cast<size_t>(ws_floats) * 4;
  return YB_OK;
}

int wgrad_grid(const WgradParams& kp) {
  const int sms = num_sms();
  return kp.total_items < sms ? kp.total_items : sms;
}

}  // namespace

}  // namespace yb

using namespace yb;

extern "C" size_t yb_conv_wgrad_workspace_bytes(const yb_wgrad_problem* problems, int n) {
  WgradParams kp;
  size_t bytes = 0;
  return wgrad_configure(problems, n, kp, &bytes) == YB_OK ? bytes : 0;
}

extern "C" int yb_conv_wgrad_config(const yb_wgrad_problem* problems, int n, int32_t* info) {
  YB_REQUIRE(info != nullptr, "conv_wgrad_config: null info array");
  WgradParams kp;
  size_t bytes = 0;
  const int rc = wgrad_configure(problems, n, kp, &bytes);
  if (rc != YB_OK) return rc;
  info[0] = kp.total_items;
  info[1] = wgrad_grid(kp);
  info[2] = static_cast<int32_t>(kSmemBytes);
  info[3] = kStages;
  info[4] = kPx;
  info[5] = kRows;
  info[6] = 64 * kMaxBlocks;
  info[7] = (kp.out_total + 255) / 256;
  for (int q = 0; q < n; ++q) {
    info[8 + 4 * q + 0] = kp.pr[q].co_tiles;
    info[8 + 4 * q + 1] = kp.pr[q].ci_tiles;
    info[8 + 4 * q + 2] = kp.pr[q].slices;
    info[8 + 4 * q + 3] = kp.pr[q].slice_len;
  }
  return YB_OK;
}

extern "C" int yb_conv_wgrad(const yb_wgrad_problem* problems, int n, void* workspace_dev, size_t workspace_bytes,
                             void* stream_) {
  WgradParams kp;
  size_t need = 0;
  int rc = wgrad_configure(problems, n, kp, &need);
  if (rc != YB_OK) return rc;
  if (workspace_dev == nullptr || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace_dev) & 15) != 0) {
    set_error("conv_wgrad: workspace of %zu bytes (16-byte aligned) needed, got %zu", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  const CUtensorMapDataType dt = problems[0].dtype == YB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  for (int q = 0; q < n && rc == YB_OK; ++q) {
    const yb_wgrad_problem& a = problems[q];
    rc = tmap_matrix(&kp.dy[q], "conv_wgrad: dy", dt, a.dy, a.Cout, a.P, a.dy_stride, 64, kPx, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc == YB_OK)
      rc = tmap_matrix(&kp.x[q], "conv_wgrad: x", dt, a.x, a.Cin, a.P, a.x_stride, 64, kPx, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  }
  if (rc != YB_OK) return rc;
  kp.ws = static_cast<float*>(workspace_dev);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool bf16 = problems[0].dtype == YB_BF16;
  const void* fn = bf16 ? reinterpret_cast<const void*>(wgrad_partial_kernel<true>)
                        : reinterpret_cast<const void*>(wgrad_partial_kernel<false>);
  YB_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBytes)));
  if (bf16) wgrad_partial_kernel<true><<<wgrad_grid(kp), kThreads, kSmemBytes, stream>>>(kp);
  else wgrad_partial_kernel<false><<<wgrad_grid(kp), kThreads, kSmemBytes, stream>>>(kp);
  YB_CHECK_CUDA(cudaGetLastError());
  int blocks = (kp.out_total + 255) / 256;
  if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
  wgrad_reduce_kernel<<<blocks, 256, 0, stream>>>(kp);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
