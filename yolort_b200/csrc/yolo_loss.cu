// YOLOv5 training loss (the reference's SetCriterion) and its gradient.  "Rule n" refers to the numbered rules in
// oracle/restate_loss.py.
//
//   flag       one thread per candidate (level, offset, anchor, target): target validation, ratio test and offset
//              conditions in the reference's fp32 arithmetic (rules 1-3)
//   scan       exclusive sum of the flags (CUB): match m's slot; the order is level, offset, anchor, target
//   emit       one thread per candidate that matched: indices, tbox, anchor (rule 4); the objectness owner of a
//              cell is its largest match index (integer atomicMax: the reference's index_put, last write wins)
//   match      one thread per match: gathered logits, CIoU and its analytic gradient, class BCE (rules 5, 7)
//   obj        BCE over every cell of every level, fixed-grid per-block partial sums (rule 6)
//   finalize   one block: per-level means in a fixed order, balance and gains (rule 8)
// backward:
//   sort key   cell of each match (stable CUB radix sort by cell keeps match order within a cell)
//   dense      every element of every level: objectness gradient on channel 4, zero elsewhere
//   sparse     one thread per matched cell: box and class gradients summed over the cell's matches in match order
#include <cub/cub.cuh>

#include "common.cuh"

namespace yb {
namespace {

constexpr int kThreads = 256;
constexpr int kObjBlocks = 256;   // blocks per level of the objectness reduction: fixed, so sums do not depend on the GPU
constexpr int kFinThreads = 512;
constexpr float kEps = 1e-7f;
constexpr float kAtanK = 0.405284734569351086f;   // 4 / pi^2

struct Match {
  int32_t level, b, a, gj, gi, cls, cell, pad;
  float tbox[4];
  float anchor[2];
  float score, lbox;
  float gbox[4];
  float lcls, pad2[3];
};
static_assert(sizeof(Match) == YB_LOSS_MATCH_INT32 * 4, "match record");

struct Level {
  const void* logits;
  int32_t dtype, H, W;
  float aw[YB_MAX_ANCHORS], ah[YB_MAX_ANCHORS];   // grid units
  int64_t cell_off;   // first cell of the level in the concatenated cell space
  int64_t cells;      // N * A * H * W
};

struct Args {
  int32_t N, L, A, nc, K, T;
  int32_t per_level;  // 5 * A * T candidates per level
  float box_gain, cls_gain, obj_gain, cls_pos, obj_pos, thresh, smooth_pos, smooth_neg, gr;
  float balance[YB_MAX_LEVELS];
  Level lv[YB_MAX_LEVELS];
};

struct Ws {
  int32_t *flags, *pos, *owner;
  Match* match;
  float* partial;   // [L][kObjBlocks]
  uint32_t *key_a, *key_b;
  int32_t *val_a, *val_b;
  void *scan_tmp, *sort_tmp;
  size_t scan_bytes, sort_bytes;
  size_t pos_off, match_off;   // byte offsets of pos and match in the workspace
};

inline size_t align_up(size_t x) { return (x + 255) & ~size_t(255); }

size_t carve(Ws& w, uint8_t* base, int64_t C, int64_t cells, int L) {
  size_t off = 0;
  auto take = [&](size_t bytes) -> uint8_t* {
    uint8_t* p = base ? base + off : nullptr;
    off += align_up(bytes);
    return p;
  };
  const size_t c1 = size_t(C) + 1;
  w.flags = reinterpret_cast<int32_t*>(take(c1 * 4));
  w.pos_off = off;
  w.pos = reinterpret_cast<int32_t*>(take(c1 * 4));
  w.owner = reinterpret_cast<int32_t*>(take(size_t(cells) * 4));
  w.match_off = off;
  w.match = reinterpret_cast<Match*>(take(size_t(C > 0 ? C : 1) * sizeof(Match)));
  w.partial = reinterpret_cast<float*>(take(size_t(L) * kObjBlocks * 4));
  const size_t cc = size_t(C > 0 ? C : 1);
  w.key_a = reinterpret_cast<uint32_t*>(take(cc * 4));
  w.key_b = reinterpret_cast<uint32_t*>(take(cc * 4));
  w.val_a = reinterpret_cast<int32_t*>(take(cc * 4));
  w.val_b = reinterpret_cast<int32_t*>(take(cc * 4));
  w.scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, w.scan_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, int(c1));
  w.scan_tmp = take(w.scan_bytes);
  w.sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, w.sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const int32_t*)nullptr, (int32_t*)nullptr, int(cc));
  w.sort_tmp = take(w.sort_bytes);
  return off;
}

__device__ __forceinline__ float load(const void* p, int dtype, int64_t i) {
  if (dtype == YB_F16) return __half2float(static_cast<const __half*>(p)[i]);
  if (dtype == YB_BF16) return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
  return static_cast<const float*>(p)[i];
}

template <typename T>
__device__ __forceinline__ T from_float(float v);
template <>
__device__ __forceinline__ float from_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float sigmoidf(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// torch's BCE-with-logits, elementwise: (1 - t) x + (1 + (pw - 1) t) (log1p(exp(-|x|)) + max(-x, 0))
__device__ __forceinline__ float bce(float x, float t, float pw) {
  const float lw = __fadd_rn(1.f, __fmul_rn(__fsub_rn(pw, 1.f), t));
  const float sp = __fadd_rn(log1pf(expf(-fabsf(x))), fmaxf(-x, 0.f));
  return __fadd_rn(__fmul_rn(__fsub_rn(1.f, t), x), __fmul_rn(lw, sp));
}
// its derivative: pw t (sigma - 1) + (1 - t) sigma
__device__ __forceinline__ float bce_grad(float x, float t, float pw) {
  const float s = sigmoidf(x);
  return __fadd_rn(__fmul_rn(__fmul_rn(pw, t), __fsub_rn(s, 1.f)), __fmul_rn(__fsub_rn(1.f, t), s));
}

// gradient weights of torch.minimum / torch.maximum for the first argument (ties split the gradient in half)
__device__ __forceinline__ float wmin(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }
__device__ __forceinline__ float wmax(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }

__device__ __forceinline__ bool target_valid(const float* t, int N, int nc, int32_t* status, bool report) {
  int bits = 0;
  if (!(t[0] >= 0.f && t[0] < float(N))) bits |= YB_LOSS_ST_IMAGE;
  if (!(t[1] >= 0.f && t[1] < float(nc))) bits |= YB_LOSS_ST_CLASS;
  if (!(isfinite(t[2]) && isfinite(t[3]) && isfinite(t[4]) && isfinite(t[5]))) bits |= YB_LOSS_ST_NONFINITE;
  if (bits && report) atomicOr(status, bits);
  return bits == 0;
}

// rule 3: v % 1 < 0.5 and v > 1 (for v > 1 the remainder is fmod, exact)
__device__ __forceinline__ bool near_low(float v) { return v > 1.f && fmodf(v, 1.f) < 0.5f; }

// ---- flag (rules 1-3) -----------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_flag_kernel(Args p, const float* __restrict__ targets,
                                                             int32_t* __restrict__ flags, int32_t* status) {
  const int64_t C = int64_t(p.L) * p.per_level;
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx > C) return;
  if (idx == C) {
    flags[C] = 0;
    return;
  }
  const int l = int(idx / p.per_level);
  const int rem = int(idx % p.per_level);
  const int o = rem / (p.A * p.T);
  const int a = (rem / p.T) % p.A;
  const int t = rem % p.T;
  float row[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) row[k] = targets[int64_t(t) * 6 + k];
  int ok = target_valid(row, p.N, p.nc, status, l == 0 && o == 0 && a == 0) ? 1 : 0;
  if (ok) {
    const Level& lv = p.lv[l];
    const float Wf = float(lv.W), Hf = float(lv.H);
    const float gw = __fmul_rn(row[4], Wf), gh = __fmul_rn(row[5], Hf);
    const float rw = __fdiv_rn(gw, lv.aw[a]), rh = __fdiv_rn(gh, lv.ah[a]);
    const float r = fmaxf(fmaxf(rw, __frcp_rn(rw)), fmaxf(rh, __frcp_rn(rh)));
    ok = r < p.thresh ? 1 : 0;
    if (ok && o > 0) {
      const float gx = __fmul_rn(row[2], Wf), gy = __fmul_rn(row[3], Hf);
      if (o == 1) ok = near_low(gx);
      else if (o == 2) ok = near_low(gy);
      else if (o == 3) ok = near_low(__fsub_rn(Wf, gx));
      else ok = near_low(__fsub_rn(Hf, gy));
    }
  }
  flags[idx] = ok;
}

// ---- emit (rule 4) --------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_emit_kernel(Args p, const float* __restrict__ targets,
                                                             const int32_t* __restrict__ flags,
                                                             const int32_t* __restrict__ pos, Match* __restrict__ out,
                                                             int32_t* __restrict__ owner) {
  const int64_t C = int64_t(p.L) * p.per_level;
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= C || !flags[idx]) return;
  const int l = int(idx / p.per_level);
  const int rem = int(idx % p.per_level);
  const int o = rem / (p.A * p.T);
  const int a = (rem / p.T) % p.A;
  const int t = rem % p.T;
  const float* row = targets + int64_t(t) * 6;
  const Level& lv = p.lv[l];
  const float Wf = float(lv.W), Hf = float(lv.H);
  const float gx = __fmul_rn(row[2], Wf), gy = __fmul_rn(row[3], Hf);
  const float gw = __fmul_rn(row[4], Wf), gh = __fmul_rn(row[5], Hf);
  const float ox = o == 1 ? 0.5f : (o == 3 ? -0.5f : 0.f);
  const float oy = o == 2 ? 0.5f : (o == 4 ? -0.5f : 0.f);
  // .long() truncates; clamping the truncated float to the grid first gives the same index for every finite value
  const int gi = int(fminf(fmaxf(truncf(__fsub_rn(gx, ox)), 0.f), Wf - 1.f));
  const int gj = int(fminf(fmaxf(truncf(__fsub_rn(gy, oy)), 0.f), Hf - 1.f));
  const int b = int(truncf(row[0]));
  const int m = pos[idx];
  Match r;
  r.level = l;
  r.b = b;
  r.a = a;
  r.gj = gj;
  r.gi = gi;
  r.cls = int(truncf(row[1]));
  const int64_t cell = lv.cell_off + ((int64_t(b) * p.A + a) * lv.H + gj) * lv.W + gi;
  r.cell = int32_t(cell);
  r.pad = 0;
  r.tbox[0] = __fsub_rn(gx, float(gi));
  r.tbox[1] = __fsub_rn(gy, float(gj));
  r.tbox[2] = gw;
  r.tbox[3] = gh;
  r.anchor[0] = lv.aw[a];
  r.anchor[1] = lv.ah[a];
  r.score = r.lbox = r.lcls = 0.f;
  r.gbox[0] = r.gbox[1] = r.gbox[2] = r.gbox[3] = 0.f;
  r.pad2[0] = r.pad2[1] = r.pad2[2] = 0.f;
  out[m] = r;
  atomicMax(owner + cell, m);
}

// ---- match (rules 5, 7) ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_match_kernel(Args p, const int32_t* __restrict__ pos,
                                                              Match* __restrict__ ms) {
  const int64_t C = int64_t(p.L) * p.per_level;
  const int m = int(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= pos[C]) return;
  Match& r = ms[m];
  const int l = r.level;
  const Level& lv = p.lv[l];
  const int M = pos[int64_t(l + 1) * p.per_level] - pos[int64_t(l) * p.per_level];
  const int64_t base = (((int64_t(r.b) * p.A + r.a) * lv.H + r.gj) * lv.W + r.gi) * p.K;
  float s[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) s[k] = sigmoidf(load(lv.logits, lv.dtype, base + k));
  // encode_single (_utils.py:26-40)
  const float px = __fsub_rn(__fmul_rn(s[0], 2.f), 0.5f), py = __fsub_rn(__fmul_rn(s[1], 2.f), 0.5f);
  const float tw = __fmul_rn(s[2], 2.f), th = __fmul_rn(s[3], 2.f);
  const float pw = __fmul_rn(__fmul_rn(tw, tw), r.anchor[0]), ph = __fmul_rn(__fmul_rn(th, th), r.anchor[1]);
  // CIoU (_utils.py:65-108), xywh -> xyxy
  const float x1 = __fsub_rn(px, pw * 0.5f), x2 = __fadd_rn(px, pw * 0.5f);
  const float y1 = __fsub_rn(py, ph * 0.5f), y2 = __fadd_rn(py, ph * 0.5f);
  const float X1 = __fsub_rn(r.tbox[0], r.tbox[2] * 0.5f), X2 = __fadd_rn(r.tbox[0], r.tbox[2] * 0.5f);
  const float Y1 = __fsub_rn(r.tbox[1], r.tbox[3] * 0.5f), Y2 = __fadd_rn(r.tbox[1], r.tbox[3] * 0.5f);
  const float iw = __fsub_rn(fminf(x2, X2), fmaxf(x1, X1)), ih = __fsub_rn(fminf(y2, Y2), fmaxf(y1, Y1));
  const float iwc = fmaxf(iw, 0.f), ihc = fmaxf(ih, 0.f);
  const float inter = __fmul_rn(iwc, ihc);
  const float w1 = __fsub_rn(x2, x1), h1 = __fadd_rn(__fsub_rn(y2, y1), kEps);
  const float w2 = __fsub_rn(X2, X1), h2 = __fadd_rn(__fsub_rn(Y2, Y1), kEps);
  const float uni = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(w1, h1), __fmul_rn(w2, h2)), inter), kEps);
  const float iou = __fdiv_rn(inter, uni);
  const float cw = __fsub_rn(fmaxf(x2, X2), fminf(x1, X1)), ch = __fsub_rn(fmaxf(y2, Y2), fminf(y1, Y1));
  const float c2 = __fadd_rn(__fadd_rn(__fmul_rn(cw, cw), __fmul_rn(ch, ch)), kEps);
  const float dx = __fsub_rn(__fsub_rn(__fadd_rn(X1, X2), x1), x2);
  const float dy = __fsub_rn(__fsub_rn(__fadd_rn(Y1, Y2), y1), y2);
  const float rho2 = __fmul_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), 0.25f);
  const float q1 = __fdiv_rn(w1, h1);
  const float d = __fsub_rn(atanf(__fdiv_rn(w2, h2)), atanf(q1));
  const float v = __fmul_rn(kAtanK, __fmul_rn(d, d));
  const float alpha = __fdiv_rn(v, __fadd_rn(__fsub_rn(v, iou), 1.0000001f));
  const float ciou = __fsub_rn(iou, __fadd_rn(__fdiv_rn(rho2, c2), __fmul_rn(v, alpha)));
  r.lbox = __fsub_rn(1.f, ciou);
  r.score = __fadd_rn(1.f - p.gr, __fmul_rn(p.gr, fmaxf(ciou, 0.f)));

  // backward of box_gain * mean(1 - CIoU), alpha constant
  const float G = -__fdiv_rn(p.box_gain, float(M));
  const float g_iou = G;
  const float g_rho2 = -__fdiv_rn(G, c2);
  const float g_c2 = __fdiv_rn(__fmul_rn(G, rho2), __fmul_rn(c2, c2));
  const float g_v = -__fmul_rn(G, alpha);
  float g_inter = __fdiv_rn(g_iou, uni);
  const float g_uni = -__fdiv_rn(__fmul_rn(g_iou, inter), __fmul_rn(uni, uni));
  g_inter -= g_uni;
  float g_w1 = __fmul_rn(g_uni, h1), g_h1 = __fmul_rn(g_uni, w1);
  const float g_d = __fmul_rn(g_v, __fmul_rn(kAtanK, 2.f * d));
  const float g_q1 = -__fdiv_rn(g_d, __fadd_rn(1.f, __fmul_rn(q1, q1)));
  g_w1 += __fdiv_rn(g_q1, h1);
  g_h1 -= __fdiv_rn(__fmul_rn(g_q1, w1), __fmul_rn(h1, h1));
  const float g_dx = __fmul_rn(g_rho2, 0.5f * dx), g_dy = __fmul_rn(g_rho2, 0.5f * dy);
  const float g_cw = __fmul_rn(g_c2, 2.f * cw), g_ch = __fmul_rn(g_c2, 2.f * ch);
  const float g_iw = iw >= 0.f ? __fmul_rn(g_inter, ihc) : 0.f;
  const float g_ih = ih >= 0.f ? __fmul_rn(g_inter, iwc) : 0.f;
  float g_x1 = -g_dx - g_w1, g_x2 = -g_dx + g_w1;
  float g_y1 = -g_dy - g_h1, g_y2 = -g_dy + g_h1;
  g_x2 += g_cw * wmax(x2, X2) + g_iw * wmin(x2, X2);
  g_x1 += -g_cw * wmin(x1, X1) - g_iw * wmax(x1, X1);
  g_y2 += g_ch * wmax(y2, Y2) + g_ih * wmin(y2, Y2);
  g_y1 += -g_ch * wmin(y1, Y1) - g_ih * wmax(y1, Y1);
  const float g_px = g_x1 + g_x2, g_pw = (g_x2 - g_x1) * 0.5f;
  const float g_py = g_y1 + g_y2, g_ph = (g_y2 - g_y1) * 0.5f;
  // encode_single backward: xy = 2 s - 0.5, wh = (2 s)^2 anchor, s = sigmoid(x)
  r.gbox[0] = __fmul_rn(__fmul_rn(g_px, 2.f), __fmul_rn(1.f - s[0], s[0]));
  r.gbox[1] = __fmul_rn(__fmul_rn(g_py, 2.f), __fmul_rn(1.f - s[1], s[1]));
  r.gbox[2] = __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(g_pw, r.anchor[0]), 2.f * tw), 2.f), __fmul_rn(1.f - s[2], s[2]));
  r.gbox[3] = __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(g_ph, r.anchor[1]), 2.f * th), 2.f), __fmul_rn(1.f - s[3], s[3]));

  float lc = 0.f;
  if (p.nc > 1) {
    for (int c = 0; c < p.nc; ++c) {
      const float t = c == r.cls ? p.smooth_pos : p.smooth_neg;
      lc += bce(load(lv.logits, lv.dtype, base + 5 + c), t, p.cls_pos);
    }
  }
  r.lcls = lc;
}

// fixed-order block sum (result valid in thread 0)
template <int kBlock>
__device__ __forceinline__ float block_sum(float v, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = 0.f;
  if (warp == 0) {
    v = lane < kBlock / 32 ? sh[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  }
  return v;
}

// ---- obj (rule 6) ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_obj_kernel(Args p, const int32_t* __restrict__ owner,
                                                            const Match* __restrict__ ms, float* __restrict__ partial) {
  __shared__ float sh[32];
  const int l = blockIdx.y;
  const Level& lv = p.lv[l];
  float acc = 0.f;
  for (int64_t c = int64_t(blockIdx.x) * kThreads + threadIdx.x; c < lv.cells; c += int64_t(kObjBlocks) * kThreads) {
    const int32_t ow = owner[lv.cell_off + c];
    const float t = ow >= 0 ? ms[ow].score : 0.f;
    acc += bce(load(lv.logits, lv.dtype, c * p.K + 4), t, p.obj_pos);
  }
  acc = block_sum<kThreads>(acc, sh);
  if (threadIdx.x == 0) partial[l * kObjBlocks + blockIdx.x] = acc;
}

// ---- finalize (rule 8) ----------------------------------------------------------------------------
__global__ void __launch_bounds__(kFinThreads) loss_finalize_kernel(Args p, const int32_t* __restrict__ pos,
                                                                    const Match* __restrict__ ms,
                                                                    const float* __restrict__ partial,
                                                                    float* __restrict__ out) {
  __shared__ float sh[32];
  float lbox = 0.f, lcls = 0.f, lobj = 0.f;
  for (int l = 0; l < p.L; ++l) {
    const int lo = pos[int64_t(l) * p.per_level], hi = pos[int64_t(l + 1) * p.per_level];
    float sb = 0.f, sc = 0.f, so = 0.f;
    for (int m = lo + threadIdx.x; m < hi; m += kFinThreads) {
      sb += ms[m].lbox;
      sc += ms[m].lcls;
    }
    for (int i = threadIdx.x; i < kObjBlocks; i += kFinThreads) so += partial[l * kObjBlocks + i];
    sb = block_sum<kFinThreads>(sb, sh);
    sc = block_sum<kFinThreads>(sc, sh);
    so = block_sum<kFinThreads>(so, sh);
    if (threadIdx.x == 0) {
      if (hi > lo) {
        lbox += sb / float(hi - lo);
        if (p.nc > 1) lcls += sc / (float(hi - lo) * float(p.nc));
      }
      const float obji = so / float(p.lv[l].cells);
      lobj += obji * p.balance[l];
      out[3 + l] = obji;
    }
  }
  if (threadIdx.x == 0) {
    out[0] = lcls * p.cls_gain;
    out[1] = lbox * p.box_gain;
    out[2] = lobj * p.obj_gain;
  }
}

// ---- backward -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_sortkey_kernel(Args p, const int32_t* __restrict__ pos,
                                                                const Match* __restrict__ ms, uint32_t* __restrict__ key,
                                                                int32_t* __restrict__ val) {
  const int64_t C = int64_t(p.L) * p.per_level;
  const int m = int(blockIdx.x) * blockDim.x + threadIdx.x;
  if (m >= C) return;
  key[m] = m < pos[C] ? uint32_t(ms[m].cell) : 0xffffffffu;
  val[m] = m;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) loss_dense_grad_kernel(Args p, int l, const int32_t* __restrict__ owner,
                                                                   const Match* __restrict__ ms,
                                                                   const float* __restrict__ grad_losses,
                                                                   T* __restrict__ out) {
  const Level& lv = p.lv[l];
  const int64_t n = lv.cells * p.K;
  // d loss_obj / d x = g_obj * obj_gain * balance / numel * bce'(x, t)
  const float coef = __fdiv_rn(__fmul_rn(__fmul_rn(grad_losses[2], p.obj_gain), p.balance[l]), float(lv.cells));
  const T* x = static_cast<const T*>(lv.logits);
  const int32_t* own = owner + lv.cell_off;
  auto one = [&](auto e, auto c) {
    float g = 0.f;
    if (e - c * p.K == 4) {
      const int32_t ow = own[c];
      const float t = ow >= 0 ? ms[ow].score : 0.f;
      g = __fmul_rn(coef, bce_grad(load(x, lv.dtype, e), t, p.obj_pos));
    }
    out[e] = from_float<T>(g);
  };
  if (n < (int64_t(1) << 31)) {   // 32-bit division by K
    const uint32_t n32 = uint32_t(n), K = uint32_t(p.K);
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n32; e += gridDim.x * blockDim.x) one(e, e / K);
  } else {
    for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += int64_t(gridDim.x) * blockDim.x)
      one(e, e / p.K);
  }
}

template <typename T>
struct Outs {
  T* p[YB_MAX_LEVELS];
};

template <typename T>
__global__ void __launch_bounds__(kThreads) loss_sparse_grad_kernel(Args p, const int32_t* __restrict__ pos,
                                                                    const uint32_t* __restrict__ key,
                                                                    const int32_t* __restrict__ val,
                                                                    const Match* __restrict__ ms,
                                                                    const float* __restrict__ grad_losses,
                                                                    Outs<T> outs) {
  const int64_t C = int64_t(p.L) * p.per_level;
  const int i = int(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= pos[C]) return;   // the keys of the matches sort first; the padding keys are all ones
  const uint32_t k = key[i];
  if (i > 0 && key[i - 1] == k) return;
  int end = i + 1;
  while (end < pos[C] && key[end] == k) ++end;
  const Match& r0 = ms[val[i]];
  const int l = r0.level;
  const Level& lv = p.lv[l];
  const int64_t base = (int64_t(k) - lv.cell_off) * p.K;
  T* out = outs.p[l];
  const float g_box = grad_losses[1];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float g = 0.f;
    for (int q = i; q < end; ++q) g += __fmul_rn(g_box, ms[val[q]].gbox[c]);
    out[base + c] = from_float<T>(g);
  }
  if (p.nc > 1) {
    const int M = pos[int64_t(l + 1) * p.per_level] - pos[int64_t(l) * p.per_level];
    const float coef = __fdiv_rn(__fmul_rn(grad_losses[0], p.cls_gain), __fmul_rn(float(M), float(p.nc)));
    for (int c = 0; c < p.nc; ++c) {
      const float x = load(lv.logits, lv.dtype, base + 5 + c);
      float g = 0.f;
      for (int q = i; q < end; ++q) {
        const float t = ms[val[q]].cls == c ? p.smooth_pos : p.smooth_neg;
        g += __fmul_rn(coef, bce_grad(x, t, p.cls_pos));
      }
      out[base + 5 + c] = from_float<T>(g);
    }
  } else {
    for (int c = 0; c < p.nc; ++c) out[base + 5 + c] = from_float<T>(0.f);
  }
}

inline unsigned blocks(int64_t n) { return unsigned((n + kThreads - 1) / kThreads); }

// host-side checks and the kernel argument block; C = candidates, cells = all cells of all levels
int prepare(const yb_yolo_loss_params* q, const yb_loss_level* levels, int64_t n_targets, Args& a, int64_t& C,
            int64_t& cells) {
  YB_REQUIRE(q && levels, "yolo_loss: null params or levels");
  YB_REQUIRE(q->n_images > 0 && q->n_levels > 0 && q->n_levels <= YB_MAX_LEVELS && q->n_anchors > 0 &&
                 q->n_anchors <= YB_MAX_ANCHORS && q->n_classes > 0,
             "yolo_loss: bad params (N %d, levels %d, anchors %d, classes %d)", q->n_images, q->n_levels, q->n_anchors,
             q->n_classes);
  YB_REQUIRE(n_targets >= 0, "yolo_loss: negative n_targets");
  a = Args{};
  a.N = q->n_images;
  a.L = q->n_levels;
  a.A = q->n_anchors;
  a.nc = q->n_classes;
  a.K = q->n_classes + 5;
  a.T = int32_t(n_targets);
  a.box_gain = q->box_gain;
  a.cls_gain = q->cls_gain;
  a.obj_gain = q->obj_gain;
  a.cls_pos = q->cls_pos;
  a.obj_pos = q->obj_pos;
  a.thresh = q->anchor_thresh;
  a.smooth_pos = q->smooth_pos;
  a.smooth_neg = q->smooth_neg;
  a.gr = q->gr;
  const int64_t per_level = int64_t(5) * a.A * n_targets;
  C = per_level * a.L;
  YB_REQUIRE(C < (int64_t(1) << 30), "yolo_loss: %lld targets are too many", (long long)n_targets);
  a.per_level = int32_t(per_level);
  cells = 0;
  for (int l = 0; l < a.L; ++l) {
    const yb_loss_level& s = levels[l];
    YB_REQUIRE(s.dtype == YB_F32 || s.dtype == YB_F16 || s.dtype == YB_BF16, "yolo_loss: level %d dtype %d", l,
               s.dtype);
    YB_REQUIRE(s.H > 0 && s.W > 0 && s.stride_px > 0.f, "yolo_loss: level %d has a bad shape", l);
    a.balance[l] = q->balance[l];
    Level& lv = a.lv[l];
    lv.logits = s.logits;
    lv.dtype = s.dtype;
    lv.H = s.H;
    lv.W = s.W;
    for (int k = 0; k < a.A; ++k) {     // rule 1: fp32 division, as torch does it
      lv.aw[k] = s.anchors_px[2 * k] / s.stride_px;
      lv.ah[k] = s.anchors_px[2 * k + 1] / s.stride_px;
      YB_REQUIRE(lv.aw[k] > 0.f && lv.ah[k] > 0.f, "yolo_loss: level %d anchor %d is not positive", l, k);
    }
    lv.cell_off = cells;
    lv.cells = int64_t(a.N) * a.A * s.H * s.W;
    cells += lv.cells;
  }
  YB_REQUIRE(cells < (int64_t(1) << 31) - 1 && cells * a.K < (int64_t(1) << 40), "yolo_loss: head outputs too large");
  return YB_OK;
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" size_t yb_yolo_loss_workspace_bytes(const yb_yolo_loss_params* params, const yb_loss_level* levels,
                                               int64_t n_targets) {
  Args a;
  int64_t C = 0, cells = 0;
  if (prepare(params, levels, n_targets, a, C, cells) != YB_OK) return 0;
  Ws w;
  return carve(w, nullptr, C, cells, a.L);
}

extern "C" int yb_yolo_loss_layout(const yb_yolo_loss_params* params, const yb_loss_level* levels, int64_t n_targets,
                                   int64_t* out) {
  Args a;
  int64_t C = 0, cells = 0;
  const int rc = prepare(params, levels, n_targets, a, C, cells);
  if (rc != YB_OK) return rc;
  YB_REQUIRE(out, "yolo_loss_layout: null out");
  Ws w;
  carve(w, nullptr, C, cells, a.L);
  out[0] = int64_t(w.match_off);
  out[1] = int64_t(w.pos_off);
  out[2] = C;
  return YB_OK;
}

extern "C" int yb_yolo_loss_forward(const yb_yolo_loss_params* params, const yb_loss_level* levels,
                                    const float* targets_dev, int64_t n_targets, float* out_losses_dev,
                                    int32_t* status_dev, void* workspace_dev, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Args a;
  int64_t C = 0, cells = 0;
  const int rc = prepare(params, levels, n_targets, a, C, cells);
  if (rc != YB_OK) return rc;
  YB_REQUIRE(out_losses_dev && status_dev && workspace_dev && (n_targets == 0 || targets_dev),
             "yolo_loss_forward: null argument");
  for (int l = 0; l < a.L; ++l) YB_REQUIRE(a.lv[l].logits, "yolo_loss_forward: level %d has no logits", l);
  Ws w;
  const size_t need = carve(w, static_cast<uint8_t*>(workspace_dev), C, cells, a.L);
  if (need > workspace_bytes) {
    set_error("yolo_loss_forward: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  YB_CHECK_CUDA(cudaMemsetAsync(w.owner, 0xff, size_t(cells) * 4, stream));
  loss_flag_kernel<<<blocks(C + 1), kThreads, 0, stream>>>(a, targets_dev, w.flags, status_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  size_t tb = w.scan_bytes;
  YB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.scan_tmp, tb, w.flags, w.pos, int(C + 1), stream));
  if (C > 0) {
    loss_emit_kernel<<<blocks(C), kThreads, 0, stream>>>(a, targets_dev, w.flags, w.pos, w.match, w.owner);
    YB_CHECK_CUDA(cudaGetLastError());
    loss_match_kernel<<<blocks(C), kThreads, 0, stream>>>(a, w.pos, w.match);
    YB_CHECK_CUDA(cudaGetLastError());
  }
  loss_obj_kernel<<<dim3(kObjBlocks, a.L), kThreads, 0, stream>>>(a, w.owner, w.match, w.partial);
  YB_CHECK_CUDA(cudaGetLastError());
  loss_finalize_kernel<<<1, kFinThreads, 0, stream>>>(a, w.pos, w.match, w.partial, out_losses_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

template <typename T>
static int backward_typed(const Args& a, const Ws& w, int64_t C, const float* grad_losses_dev,
                          void* const* grad_out_levels, cudaStream_t stream) {
  for (int l = 0; l < a.L; ++l) {
    const int64_t n = a.lv[l].cells * a.K;
    const unsigned grid = unsigned(std::min<int64_t>(blocks(n), int64_t(num_sms()) * 16));
    loss_dense_grad_kernel<T><<<grid, kThreads, 0, stream>>>(a, l, w.owner, w.match, grad_losses_dev,
                                                             static_cast<T*>(grad_out_levels[l]));
    YB_CHECK_CUDA(cudaGetLastError());
  }
  if (C > 0) {
    Outs<T> outs = {};
    for (int l = 0; l < a.L; ++l) outs.p[l] = static_cast<T*>(grad_out_levels[l]);
    loss_sparse_grad_kernel<T><<<blocks(C), kThreads, 0, stream>>>(a, w.pos, w.key_b, w.val_b, w.match,
                                                                   grad_losses_dev, outs);
    YB_CHECK_CUDA(cudaGetLastError());
  }
  return YB_OK;
}

extern "C" int yb_yolo_loss_backward(const yb_yolo_loss_params* params, const yb_loss_level* levels,
                                     int64_t n_targets, const float* grad_losses_dev, void* const* grad_out_levels,
                                     void* workspace_dev, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Args a;
  int64_t C = 0, cells = 0;
  const int rc = prepare(params, levels, n_targets, a, C, cells);
  if (rc != YB_OK) return rc;
  YB_REQUIRE(grad_losses_dev && grad_out_levels && workspace_dev, "yolo_loss_backward: null argument");
  for (int l = 0; l < a.L; ++l) {
    YB_REQUIRE(grad_out_levels[l] && a.lv[l].logits, "yolo_loss_backward: level %d has no output", l);
    YB_REQUIRE(levels[l].dtype == levels[0].dtype, "yolo_loss_backward: levels must share a dtype");
  }
  Ws w;
  const size_t need = carve(w, static_cast<uint8_t*>(workspace_dev), C, cells, a.L);
  if (need > workspace_bytes) {
    set_error("yolo_loss_backward: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  if (C > 0) {
    loss_sortkey_kernel<<<blocks(C), kThreads, 0, stream>>>(a, w.pos, w.match, w.key_a, w.val_a);
    YB_CHECK_CUDA(cudaGetLastError());
    size_t tb = w.sort_bytes;
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tb, w.key_a, w.key_b, w.val_a, w.val_b, int(C), 0, 32,
                                                  stream));
  }
  switch (levels[0].dtype) {
    case YB_F16: return backward_typed<__half>(a, w, C, grad_losses_dev, grad_out_levels, stream);
    case YB_BF16: return backward_typed<__nv_bfloat16>(a, w, C, grad_losses_dev, grad_out_levels, stream);
    default: return backward_typed<float>(a, w, C, grad_losses_dev, grad_out_levels, stream);
  }
}
