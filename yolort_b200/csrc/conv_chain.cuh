// Chained pointwise tail (yb_conv_chain): parameters shared by the two convolution kernels and the host-side set-up.
//
// After the first convolution's epilogue has written its output boxes into the swizzled staging buffers (the layout a
// TMA store reads AND the K-major layout a wgmma operand descriptor expresses), the two consumer warpgroups multiply
// those boxes with the resident tail weights into their (now drained) accumulator registers; a second epilogue pass
// stores the tail's output.  Reference chains: yolort/v5/models/common.py:94-116 (Bottleneck cv1 after the previous conv),
// :149-173 (C3: cv1||cv2 -> m.0.cv1, m.last.cv2 -> cv3 over the concat).
#pragma once
#include "conv_epilogue.cuh"
#include "host_sm90.h"

namespace yb {

struct ChainParams {
  int on;
  int n2;                 // accumulator columns of the tail GEMM (Cout_pad of the tail rounded up to a power of two)
  int own_chunks;         // own output boxes that feed the tail (1 or 2); box b sits in staging buffer b of the group
  int own_row_bytes;      // row pitch of an own box (= store_cols * 2 of the first convolution)
  int extra_on;           // one more operand chunk, TMA-loaded per tile into staging buffer `own_chunks`
  int extra_row_bytes;    // = kc * 2
  uint32_t extra_bytes;   // bytes of one extra chunk (128 rows)
  int ksteps;             // K=16 steps per chunk (kc / 16, kc = channels per chunk)
  int store_first;        // the first convolution's output is also written to memory
  uint32_t w2_sub_bytes;  // bytes reserved per weight chunk [n2][kc] (1024-aligned)
  int w2_chunks;          // own_chunks + extra_on
  int w2_row_bytes;       // kc * 2
  const float* bias2;
  int bias2_len;
  EpilogueParams ep2;     // Cout / act of the tail (no residual)
};

// Host side: validates a yb_conv_chain against the first convolution's tiling and fills ChainParams.
//   block_n / n_tiles / store_cols1: N tiling and TMA-store box width of the first convolution.
// Returns nullptr on success, else a static reason string.
inline const char* chain_setup(const yb_op_desc& d, int block_n, int n_tiles, int store_cols1, bool allow_extra,
                               ChainParams* cp) {
  const yb_conv_chain& c = *d.chain;
  if (d.decode != nullptr) return "fused decode and a chained tail exclude each other";
  if (d.act >= YB_ACT_HARDSWISH || c.act >= YB_ACT_HARDSWISH) return "r3.1 activations are not chained";
  if (c.act < YB_ACT_NONE) return "bad tail activation";
  if (!c.weight || !c.bias || !c.out) return "tail without weight/bias/out";
  if (n_tiles != 1) return "the first convolution must have a single N tile";
  if (c.own_C <= 0 || c.own_C > d.Cout) return "own_C outside the first convolution's output";
  const int kc = c.own_C >= 64 ? 64 : c.own_C;
  if (kc != 16 && kc != 32 && kc != 64) return "own_C must be 16, 32, 64 or 128";
  if (c.own_C % kc) return "own_C must be a multiple of its chunk width";
  const int own_chunks = c.own_C / kc;
  if (own_chunks > 2) return "at most two own chunks (own_C <= 128)";
  const int n1_boxes = block_n / store_cols1;
  if (n1_boxes > 2) return "the first convolution's tile must fit two staging boxes";
  if (own_chunks == 2 && store_cols1 != 64) return "two own chunks need 64-column boxes";
  if (kc > store_cols1) return "own chunk wider than a staging box";
  const int extra_on = c.extra != nullptr ? 1 : 0;
  if (extra_on) {
    if (!allow_extra) return "an extra operand needs the halo-patch kernel (rectangular tiles)";
    if (c.extra_C != kc) return "extra_C must equal the own chunk width";
    if (own_chunks != 1) return "extra operand with two own chunks";
    if ((reinterpret_cast<uintptr_t>(c.extra) & 15) || c.extra_cstride % 8 || c.extra_cstride < c.extra_C) return "extra operand alignment";
  } else if (c.extra_C != 0) {
    return "extra_C without an extra pointer";
  }
  if (c.K_pad != (own_chunks + extra_on) * kc) return "K_pad must equal own_C + extra_C";
  if (c.Cout_pad % 16 || c.Cout_pad < c.Cout || c.Cout_pad > 256 || c.Cout % 8) return "tail Cout/Cout_pad";
  if (c.out_cstride % 8 || c.out_cstride < c.Cout) return "tail out_cstride";
  if ((reinterpret_cast<uintptr_t>(c.out) & 15) || (reinterpret_cast<uintptr_t>(c.weight) & 15)) return "tail tensors must be 16-byte aligned";
  const int n2 = mma_n(c.Cout_pad);
  cp->on = 1;
  cp->n2 = n2;
  cp->own_chunks = own_chunks;
  cp->own_row_bytes = store_cols1 * 2;
  cp->extra_on = extra_on;
  cp->extra_row_bytes = kc * 2;
  cp->extra_bytes = 128u * kc * 2;
  cp->ksteps = kc / 16;
  cp->store_first = c.store_first ? 1 : 0;
  cp->w2_sub_bytes = (static_cast<uint32_t>(n2 * kc * 2) + 1023u) & ~1023u;
  cp->w2_chunks = own_chunks + extra_on;
  cp->w2_row_bytes = kc * 2;
  cp->bias2 = c.bias;
  cp->bias2_len = c.Cout_pad;
  cp->ep2.Cout = c.Cout;
  cp->ep2.act = c.act;
  cp->ep2.is_bf16 = d.dtype == YB_BF16;
  cp->ep2.residual = nullptr;
  cp->ep2.res_cstride = 0;
  return nullptr;
}

// TMA-store box width of the tail's output (the kernels are instantiated for 64 and 32).
__host__ __device__ inline int chain_store2_cols(int n2) { return (n2 % 64 == 0) ? 64 : ((n2 % 32 == 0) ? 32 : 16); }

}  // namespace yb
