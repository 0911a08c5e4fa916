// Multi-head scaled-dot-product attention on the Hopper tensor cores (wgmma), flash style.
//
//   O_h = softmax(Q_h K_h^T / sqrt(64)) V_h          per image and head, no mask, over the L = H*W tokens of an image
//
// Replaces the attention of nn.MultiheadAttention inside the reference's TransformerLayer
// (yolort/v5/models/common.py:308-331, C3TR at :360-367): the in-projections and out_proj around it are ordinary 1x1
// convolutions of the plan.  Q, K and V are one packed NHWC view [q | k | v] (3E channels per token); head h reads
// channels h*64 .. h*64+63 of each third and writes channels h*64 .. of the E-channel output view.
//
// One CTA per (64-query tile, head, image), 160 threads:
//   warps 0-3 (consumer warpgroup): S = Q K^T with wgmma (Q and K both K-major from shared memory, 128-byte swizzle),
//             online softmax in fp32 on the accumulator fragment (running max and sum per row, exp2 with
//             log2(e)/sqrt(d) folded into one multiply), then O += P V with P converted in registers into the A
//             fragment of the next wgmma and V read as an MN-major B operand.  One division per row at the end; O is
//             staged in shared memory (swizzled) and stored by TMA, which clips the query rows past L.
//   warp 4 (producer): TMA loads of the Q tile once and of the K / V tiles of 64 keys through a ring of mbarrier
//             stages.  One 3-D tensor map {channel, token, image} over the qkv view serves all three: the loads of an
//             image never cross into the next one, and tokens past L are zero-filled.  Zero-filled keys are not a
//             mask: their scores are set to -inf in the last tile.
// No L x L tensor ever reaches memory, there are no atomics (deterministic), and nothing is allocated or synchronised
// on the host (graph-capturable).
#include "common.cuh"
#include "conv_sm90.h"

namespace yb {

namespace {

constexpr int kHeadDim = 64;
constexpr int kBlockQ = 64;                        // query rows per CTA (one consumer warpgroup)
constexpr int kBlockKV = 64;                       // keys per pipeline stage
constexpr int kStages = 3;
constexpr int kThreads = 128 + 32;                 // consumer warpgroup + producer warp
constexpr uint32_t kTileBytes = kBlockKV * kHeadDim * 2;   // 64 rows x 128 bytes (also the Q tile)
constexpr size_t kSmemBytes = 1024 + kTileBytes * (1 + 2 * kStages);   // Q (then O staging) + K/V ring, 1 KB alignment

struct AttnParams {
  int L;        // tokens per image
  int E;        // channels per third of the qkv view (heads * 64)
  float scale_log2;
};

// O[64 x 64] (+)= P[64 x 16] * V[16 x 64]: P from registers (the f16/bf16 A fragment), V an MN-major B operand.
template <bool kBf16>
__device__ __forceinline__ void wgmma_n64_rs(float* d, const uint32_t* a, uint64_t db) {
  if constexpr (!kBf16) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
  } else {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
  }
}

template <bool kBf16>
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  if constexpr (kBf16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// grid (query tiles, heads, images)
template <bool kBf16>
__global__ void __launch_bounds__(kThreads)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_out,
                       const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages];
  __shared__ __align__(8) uint64_t empty_bar[kStages];
  __shared__ __align__(8) uint64_t q_full;

  // 128-byte swizzled tiles need 1024-byte alignment
  uint8_t* q_tile = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* kv = q_tile + kTileBytes;   // stage s: K at kv + 2s*kTileBytes, V right after it

  const int q0 = blockIdx.x * kBlockQ;
  const int head = blockIdx.y;
  const int img = blockIdx.z;
  const int n_kv = (p.L + kBlockKV - 1) / kBlockKV;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_out);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);
    }
    mbar_init(&q_full, 1);
    mbar_fence_init();
  }
  __syncthreads();
  // Programmatic dependent launch: the qkv view is written by the previous kernel, and the output view may still be
  // read by an earlier one.  Every thread waits before it touches either.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp == 4) {
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    const int cq = head * kHeadDim, ck = p.E + head * kHeadDim, cv = 2 * p.E + head * kHeadDim;
    if (YB_ELECT()) {
      mbar_expect_tx(&q_full, kTileBytes);
      tma_load_3d(&tmap_qkv, &q_full, q_tile, cq, q0, img);
    }
    for (int t = 0; t < n_kv; ++t) {
      const int s = t % kStages;
      mbar_wait(&empty_bar[s], ((t / kStages) & 1) ^ 1);
      if (YB_ELECT()) {
        uint8_t* k_dst = kv + 2 * s * kTileBytes;
        mbar_expect_tx(&full_bar[s], 2 * kTileBytes);
        tma_load_3d(&tmap_qkv, &full_bar[s], k_dst, ck, t * kBlockKV, img);
        tma_load_3d(&tmap_qkv, &full_bar[s], k_dst + kTileBytes, cv, t * kBlockKV, img);
      }
    }
    return;
  }

  // ===================== consumer warpgroup =====================
  // Accumulator fragment of m64nNk16 (N = 64 here): register 4j+i holds row 16*warp + lane/4 (+8 for i >= 2) and
  // column 8j + 2*(lane%4) + (i&1).
  const int r_lo = warp * 16 + (lane >> 2);
  const int q2 = 2 * (lane & 3);
  const uint32_t kmaj_hi = desc_hi(128, 1024);
  // V is read MN-major: rows of 128 bytes are keys, the 64 head-dim columns run along them; a K=16 step spans two
  // 8-key swizzle atoms 1024 bytes apart (the stride field of an MN-major descriptor; the leading-byte field would step
  // to the next 64 columns, which a 64-wide tile does not have, and is set to the same value).
  const uint32_t vmaj_hi = static_cast<uint32_t>((1024u >> 4) | (1ull << 30));   // SBO = 1024, 128-byte swizzle
  const uint32_t vmaj_lbo = (1024u >> 4) << 16;
  const uint32_t q_lo = smem_lo16(q_tile);

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};

  mbar_wait(&q_full, 0);
  for (int t = 0; t < n_kv; ++t) {
    const int s = t % kStages;
    mbar_wait(&full_bar[s], (t / kStages) & 1);
    const uint32_t k_lo = smem_lo16(kv + 2 * s * kTileBytes);
    const uint32_t v_lo = k_lo + (kTileBytes >> 4);

    // ---- S = Q K^T: 64 x 64, K = 64 head dims in four K=16 steps ----
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHeadDim / 16; ++k)
      wgmma_mma<kBf16, 64>(sc, desc_lohi(q_lo + 2 * k, kmaj_hi), desc_lohi(k_lo + 2 * k, kmaj_hi), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc<32>(sc);

    // ---- online softmax on the fragment (rows r_lo and r_lo + 8; a quad of lanes shares each row) ----
    const int key0 = t * kBlockKV;
    if (key0 + kBlockKV > p.L) {   // last tile: zero-filled keys past L are masked
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (key0 + 8 * j + q2 + (i & 1) >= p.L) sc[4 * j + i] = -INFINITY;
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * r], sc[4 * j + 2 * r + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[r], mx * p.scale_log2);   // every tile holds at least one unmasked key
      alpha[r] = fast_exp2(m_run[r] - m_new);                     // 0 on the first tile (m_run = -inf)
      m_run[r] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float e = fast_exp2(fmaf(sc[4 * j + 2 * r + i], p.scale_log2, -m_new));
          sc[4 * j + 2 * r + i] = e;
          sum += e;
        }
      }
      l_run[r] = l_run[r] * alpha[r] + sum;   // per-thread partial sum over its columns, reduced across the quad at the end
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j + 0] *= alpha[0];
      o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1];
      o[4 * j + 3] *= alpha[1];
    }

    // ---- O += P V: P's accumulator columns 16k .. 16k+15 are exactly the A fragment of K step k ----
    uint32_t pa[16];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      pa[4 * k + 0] = pack2<kBf16>(sc[8 * k + 0], sc[8 * k + 1]);
      pa[4 * k + 1] = pack2<kBf16>(sc[8 * k + 2], sc[8 * k + 3]);
      pa[4 * k + 2] = pack2<kBf16>(sc[8 * k + 4], sc[8 * k + 5]);
      pa[4 * k + 3] = pack2<kBf16>(sc[8 * k + 6], sc[8 * k + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockKV / 16; ++k)
      wgmma_n64_rs<kBf16>(o, pa + 4 * k, desc_lohi((v_lo + k * (2048 >> 4)) | vmaj_lbo, vmaj_hi));
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc<32>(o);
    if (threadIdx.x == 0) mbar_arrive(&empty_bar[s]);   // both MMAs that read stage s have completed
  }

  // ---- epilogue: O / l -> f16/bf16 -> swizzled staging in the Q tile (dead now) -> TMA store ----
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[r] = 1.f / l;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r_lo + 8 * r;
      // 128-byte swizzle: 16-byte chunk j of row `row` sits at chunk j ^ (row % 8)
      uint8_t* dst = q_tile + row * 128 + ((j ^ (row & 7)) << 4) + q2 * 2;
      *reinterpret_cast<uint32_t*>(dst) = pack2<kBf16>(o[4 * j + 2 * r] * inv[r], o[4 * j + 2 * r + 1] * inv[r]);
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 128);
  if (threadIdx.x == 0) {
    tma_store_3d(&tmap_out, q_tile, head * kHeadDim, q0, img);
    tma_store_commit();
    tma_store_wait_all<0>();
  }
}

}  // namespace

struct AttentionOp {
  CUtensorMap tmap_qkv, tmap_out;
  AttnParams p;
  dim3 grid;
  bool bf16;
};

int attention_configure_check(const yb_op_desc& d) {
  YB_REQUIRE(d.dtype == YB_F16 || d.dtype == YB_BF16, "attention: dtype must be f16 or bf16");
  YB_REQUIRE(d.weight == nullptr && d.bias == nullptr && d.residual == nullptr && d.decode == nullptr && d.chain == nullptr,
             "attention: weight, bias, residual, decode and chain must be NULL");
  YB_REQUIRE(d.act == YB_ACT_NONE && d.reserved == 0, "attention: act and reserved must be 0");
  YB_REQUIRE(d.N >= 1 && d.H >= 1 && d.W >= 1, "attention: empty sequence (N=%d H=%d W=%d)", d.N, d.H, d.W);
  YB_REQUIRE(d.Ho == d.H && d.Wo == d.W, "attention: output extent (%d,%d) must equal the input extent (%d,%d)", d.Ho,
             d.Wo, d.H, d.W);
  const long long L = static_cast<long long>(d.H) * d.W;
  YB_REQUIRE(L < (1ll << 31) && static_cast<long long>(d.N) <= 65535, "attention: sequence or batch too large");
  YB_REQUIRE(d.ksize >= 1, "attention: ksize holds the head count, got %d", d.ksize);
  YB_REQUIRE(d.Cout % d.ksize == 0, "attention: E=%d is not a multiple of the %d heads", d.Cout, d.ksize);
  YB_REQUIRE(d.Cout / d.ksize == kHeadDim, "attention: head_dim must be %d, got %d", kHeadDim, d.Cout / d.ksize);
  YB_REQUIRE(d.Cin == 3 * d.Cout, "attention: the input holds [q | k | v]: Cin must be 3E=%d, got %d", 3 * d.Cout, d.Cin);
  YB_REQUIRE(d.Cin % 8 == 0 && d.in_cstride % 8 == 0 && d.in_cstride >= d.Cin,
             "attention: Cin/in_cstride must be multiples of 8 with in_cstride >= Cin, got %d/%d", d.Cin, d.in_cstride);
  YB_REQUIRE(d.Cout % 8 == 0 && d.out_cstride % 8 == 0 && d.out_cstride >= d.Cout,
             "attention: Cout/out_cstride must be multiples of 8 with out_cstride >= Cout, got %d/%d", d.Cout, d.out_cstride);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(d.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0,
             "attention: tensors must be 16-byte aligned");
  return YB_OK;
}

int attention_op_create(const yb_op_desc& d, AttentionOp** out) {
  int rc = attention_configure_check(d);
  if (rc != YB_OK) return rc;
  AttentionOp* op = new AttentionOp();
  const long long L = static_cast<long long>(d.H) * d.W;
  op->bf16 = d.dtype == YB_BF16;
  op->p.L = static_cast<int>(L);
  op->p.E = d.Cout;
  op->p.scale_log2 = 1.4426950408889634f / 8.f;   // log2(e) / sqrt(64)
  op->grid = dim3(static_cast<unsigned>((L + kBlockQ - 1) / kBlockQ), static_cast<unsigned>(d.ksize), static_cast<unsigned>(d.N));
  const CUtensorMapDataType dt = op->bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const cuuint32_t box[3] = {kHeadDim, kBlockKV, 1};
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(d.Cin), static_cast<cuuint64_t>(L), static_cast<cuuint64_t>(d.N)};
  rc = tmap_tiled(&op->tmap_qkv, "attention q | k | v", dt, d.in, 3, dims, d.in_cstride, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  if (rc == YB_OK) {
    const cuuint64_t odims[3] = {static_cast<cuuint64_t>(d.Cout), static_cast<cuuint64_t>(L), static_cast<cuuint64_t>(d.N)};
    rc = tmap_tiled(&op->tmap_out, "attention output", dt, d.out, 3, odims, d.out_cstride, box, CU_TENSOR_MAP_L2_PROMOTION_NONE);
  }
  if (rc != YB_OK) {
    delete op;
    return rc;
  }
  cudaError_t e = op->bf16 ? cudaFuncSetAttribute(attention_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  static_cast<int>(kSmemBytes))
                           : cudaFuncSetAttribute(attention_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  static_cast<int>(kSmemBytes));
  if (e != cudaSuccess) {
    set_error("attention: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    delete op;
    return YB_ERR_CUDA;
  }
  *out = op;
  return YB_OK;
}

int attention_op_launch(const AttentionOp* op, cudaStream_t stream) {
  YB_CHECK_CUDA(launch_pdl(op->bf16 ? attention_wgmma_kernel<true> : attention_wgmma_kernel<false>, op->grid, dim3(kThreads),
                           kSmemBytes, stream, op->tmap_qkv, op->tmap_out, op->p));
  return YB_OK;
}

void attention_op_destroy(AttentionOp* op) { delete op; }

}  // namespace yb
