// Post-processing: anchor decode + multi-label threshold + batched NMS + top-k + box rescale.
//
// Replaces PostProcess.forward (yolort/models/box_head.py:388-429):
//   _concat_pred_logits  :328-348  sigmoid, det_utils.decode_single (_utils.py:43-62)
//   _decode_pred_logits  :351-360  scores = cls * obj ; box_convert(cxcywh -> xyxy)
//   torch.where(scores > thr) :418 row-major (anchor, class) candidates -- multi-label
//   torchvision.ops.batched_nms :422 (coordinate-offset trick or per-class, by numel) ; keep[:max_det]
// and YOLOTransform.postprocess / scale_coords (yolort/models/transform.py:332-367).
//
// Two kernels per batch (plus a counter reset), no host round trip:
//   1. decode.  decode_rows_kernel for the plan's NHWC head buffers (one 512-byte row per pixel): a warp copies the
//      rows of its 32 pixels into shared memory, lane = pixel tests the objectness of its anchors (an anchor whose
//      sigmoid(obj) <= thr cannot produce a candidate: cls < 1), the (pixel, anchor) pairs that passed are compacted
//      across the warp and lane q scans the classes of pair q; decode_candidates_kernel (one thread per anchor) for any
//      other layout (the reference's [N,A,H,W,K], fp32 logits).  Survivors decode the box once (fp32, unfused ops in the
//      reference's order), write it to a dense per-anchor array and append one 64-bit sort key per (anchor, class) over
//      threshold:
//          key = ~orderable(score) << 32 | (anchor * nc + class)
//      so ascending key order == score descending, ties in row-major candidate order (what a stable
//      sort of the reference's candidate list gives).
//   2. nms_image_kernel -- one 512-thread CTA per image: sorts the image's keys (bitonic network on keys held in
//      registers, up to 4096; in-CTA LSD radix sort through global memory above that), then the greedy sweep:
//      candidates are consumed 512 at a time; each thread tests its candidate against the kept list (<= max_det boxes
//      in shared memory), the survivors' suppression bit-matrix is built with the (row, word) pairs dealt out evenly,
//      and they are resolved in order 32 at a time from registers.  The sweep stops at max_det keeps, exactly like
//      keep[:detections_per_img].
// IoU arithmetic mirrors torchvision's CPU nms kernel in fp32 with explicit non-fused operations so the
// keep set is bit-identical on identical inputs.
#include <climits>
#include <type_traits>

#include "common.cuh"
#include "decode_common.cuh"

namespace yb {
namespace {

constexpr int kNmsThreads = 512;
constexpr int kSweep = 512;       // candidates consumed per sweep round (== threads)
constexpr int kMaxLabelMasks = 256; // per-class survivor bit-masks are used up to this many classes
constexpr int kSmallSort = 4096;  // keys sorted in shared memory

template <typename T>
__device__ __forceinline__ float ld_logit(const void* base, long long off);
template <>
__device__ __forceinline__ float ld_logit<float>(const void* base, long long off) {
  return __ldg(static_cast<const float*>(base) + off);
}
template <>
__device__ __forceinline__ float ld_logit<__half>(const void* base, long long off) {
  return __half2float(__ldg(static_cast<const __half*>(base) + off));
}
template <>
__device__ __forceinline__ float ld_logit<__nv_bfloat16>(const void* base, long long off) {
  return __bfloat162float(static_cast<const __nv_bfloat16*>(base)[off]);
}

struct DecodeParams {
  static constexpr int kLevels = YB_MAX_LEVELS;
  yb_head_level lvl[YB_MAX_LEVELS];
  int lvl_start[YB_MAX_LEVELS + 1];  // first flat anchor index of each level
  int pix_start[YB_MAX_LEVELS + 1];  // first flat PIXEL index of each level (row kernel)
  int n_images, n_levels, n_anchors, n_classes;
  int anchors_per_image;
  float score_thresh;
  long long cap_per_image;
};

// Multi-pass (test-time augmentation) decode: the kept level slices of up to YB_TTA_MAX_PASSES passes, in the order the
// reference concatenates them (v5/models/yolo.py:161-162), each with its pass's descale (:180-185).
constexpr int kTtaLevels = YB_TTA_MAX_PASSES * YB_MAX_LEVELS;
struct TtaDecodeParams {
  static constexpr int kLevels = kTtaLevels;
  yb_head_level lvl[kTtaLevels];
  int lvl_start[kTtaLevels + 1];
  int pix_start[kTtaLevels + 1];
  int n_images, n_levels, n_anchors, n_classes;
  int anchors_per_image;
  float score_thresh;
  long long cap_per_image;
  float scale[kTtaLevels];     // the level's pass scale s: (cx, cy, w, h) /= s
  float flip_w[kTtaLevels];    // mirrored pass: cx = Wb - cx after the descale; 0: not mirrored
  int flip[kTtaLevels];
};

// workspace carve-up (device)
struct Workspace {
  uint64_t* keys_a;    // [n][cap]
  uint64_t* keys_b;    // [n][cap]
  float4* boxes;       // [n][anchors_per_image]
  int* img_count;      // [n]
  int* img_maxc;       // [n] ordered-int max coordinate over candidate boxes
  long long* status;   // [4] scratch status block (used when the caller passes none)
};

// One thread tests one anchor's objectness; the warp then scans the classes of every passing anchor
// cooperatively (lane k <-> class k, coalesced 2-byte/4-byte loads) and appends candidates with one
// aggregated atomic per 32 classes.
template <typename T>
__global__ void decode_candidates_kernel(const __grid_constant__ DecodeParams p, Workspace ws) {
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(p.n_images) * p.anchors_per_image;
  const int lane = threadIdx.x & 31;
  bool pass = false;
  int img = 0, anchor = 0, l = 0, x = 0, y = 0, a = 0;
  long long off = 0;
  float obj = 0.f;
  if (gid < total) {
    img = static_cast<int>(gid / p.anchors_per_image);
    anchor = static_cast<int>(gid - static_cast<long long>(img) * p.anchors_per_image);
#pragma unroll
    for (int i = 1; i < YB_MAX_LEVELS; ++i)
      if (i < p.n_levels && anchor >= p.lvl_start[i]) l = i;
    const yb_head_level& L = p.lvl[l];
    int r = anchor - p.lvl_start[l];
    x = r % L.W;
    r /= L.W;
    y = r % L.H;
    a = r / L.H;
    off = img * L.stride_n + a * L.stride_a + y * L.stride_y + x * L.stride_x;
    obj = sigmoidf_ref(ld_logit<T>(L.logits, off + 4));
    pass = obj > p.score_thresh;  // score = cls*obj <= obj, so failing anchors cannot yield candidates
  }
  uint32_t todo = __ballot_sync(0xffffffffu, pass);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const int s_img = __shfl_sync(0xffffffffu, img, src);
    const int s_anchor = __shfl_sync(0xffffffffu, anchor, src);
    const int s_l = __shfl_sync(0xffffffffu, l, src);
    const int s_x = __shfl_sync(0xffffffffu, x, src);
    const int s_y = __shfl_sync(0xffffffffu, y, src);
    const int s_a = __shfl_sync(0xffffffffu, a, src);
    const long long s_off = __shfl_sync(0xffffffffu, off, src);
    const float s_obj = __shfl_sync(0xffffffffu, obj, src);
    const yb_head_level& L = p.lvl[s_l];
    bool any = false;
    for (int k0 = 0; k0 < p.n_classes; k0 += 32) {
      const int k = k0 + lane;
      float score = 0.f;
      bool cand = false;
      if (k < p.n_classes) {
        const float cls = sigmoidf_ref(ld_logit<T>(L.logits, s_off + 5 + k));
        score = __fmul_rn(cls, s_obj);
        cand = score > p.score_thresh;
      }
      const uint32_t cm = __ballot_sync(0xffffffffu, cand);
      if (cm == 0) continue;
      any = true;
      int base = 0;
      if (lane == 0) base = atomicAdd(&ws.img_count[s_img], __popc(cm));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (cand) {
        const int slot = base + __popc(cm & ((1u << lane) - 1u));
        if (slot < p.cap_per_image) {
          const uint64_t key = (static_cast<uint64_t>(orderable_desc(score)) << 32) |
                               static_cast<uint32_t>(s_anchor * p.n_classes + k);
          ws.keys_a[static_cast<long long>(s_img) * p.cap_per_image + slot] = key;
        }
      }
    }
    if (any) {
      // box of this anchor: lanes 0..3 fetch tx,ty,tw,th
      float t = 0.f;
      if (lane < 4) t = sigmoidf_ref(ld_logit<T>(L.logits, s_off + lane));
      const float sx = __shfl_sync(0xffffffffu, t, 0), sy = __shfl_sync(0xffffffffu, t, 1);
      const float sw = __shfl_sync(0xffffffffu, t, 2), sh = __shfl_sync(0xffffffffu, t, 3);
      if (lane == 0) {
        // _utils.py:59-60 in the reference's op order: (y*2 - 0.5 + grid) * stride ; (y*2)**2 * anchor
        const float cx = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sx, 2.0f), 0.5f), static_cast<float>(s_x)), L.stride_px);
        const float cy = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(sy, 2.0f), 0.5f), static_cast<float>(s_y)), L.stride_px);
        const float tw = __fmul_rn(sw, 2.0f), th = __fmul_rn(sh, 2.0f);
        const float w = __fmul_rn(__fmul_rn(tw, tw), L.anchors_px[2 * s_a]);
        const float h = __fmul_rn(__fmul_rn(th, th), L.anchors_px[2 * s_a + 1]);
        // torchvision box_convert cxcywh -> xyxy
        const float hw = __fmul_rn(0.5f, w), hh = __fmul_rn(0.5f, h);
        const float4 b = make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
        ws.boxes[static_cast<long long>(s_img) * p.anchors_per_image + s_anchor] = b;
        atomicMax(&ws.img_maxc[s_img], float_to_ordered_int(fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w))));
      }
    }
  }
}

// Row variant for the plan's NHWC head buffers (channel a*K + k, row = one pixel's A*K logits, <= 512 bytes,
// 16-byte aligned): HBM-bound, so the point is to fetch every byte exactly once, coalesced, to spend almost no
// instructions per pixel, and to keep the per-image counters out of the way.  A block takes 128 consecutive pixels
// of ONE image; each warp copies the rows of its 32 pixels into shared memory with cp.async (per row one 512-byte
// fully coalesced request, 16 KB in flight per warp, no register staging), then LANE l OWNS PIXEL l: it tests the
// objectness of its pixel's anchors and scans the classes of those that pass, 32 pixels wide, out of shared memory, a
// raw-logit pre-test sparing the exact sigmoid for almost every class.  Candidates are
// collected in a block-local list and appended to the image's key arena with ONE global atomic per block: with an
// atomic per candidate group the kernel is bound by ~2 000 same-address L2 atomics per image.
// Arithmetic, candidate keys and the dense box array are those of the kernel above.
constexpr int kRowPixels = 32;       // pixels per warp
constexpr int kRowWarps = 4;         // warps per block
constexpr int kRowMaxBytes = 512;    // longest row handled (A*K 16-bit logits padded to a multiple of 8)
constexpr int kRowPitch = kRowMaxBytes + 16;   // shared-memory row pitch: 132 words -> lanes spread over 8 banks
constexpr int kRowList = 512;        // block-local candidate list (entries beyond it fall back to global atomics)
constexpr int kRowPairs = kRowPixels * YB_MAX_ANCHORS;   // per-warp list of (pixel, anchor) pairs that passed objectness

// bit positions in the row kernel's (pixel, anchor) pair word: px | py << 10 | level << kLv | anchor << kAnchor | lane << kLane
template <typename Params>
struct PairBits {
  static constexpr int kLv = 20, kLvMask = 3, kAnchor = 22, kLane = 24;
};
template <>
struct PairBits<TtaDecodeParams> {   // 12 level slices: 4 bits of level
  static constexpr int kLv = 27, kLvMask = 15, kAnchor = 20, kLane = 22;
};

// candidate index (key low word) and box of one anchor: the single-pass kernel's, and the multi-pass kernel's (unsigned
// index: anchors x classes may exceed 2^31; box descaled / un-mirrored before the corner conversion)
__device__ __forceinline__ uint32_t candidate_index(const DecodeParams& p, int anchor, int k) {
  return static_cast<uint32_t>(anchor * p.n_classes + k);
}
__device__ __forceinline__ uint32_t candidate_index(const TtaDecodeParams& p, int anchor, int k) {
  return static_cast<uint32_t>(anchor) * static_cast<uint32_t>(p.n_classes) + static_cast<uint32_t>(k);
}
__device__ __forceinline__ float4 pass_box(const DecodeParams&, int, float sx, float sy, float sw, float sh, int x, int y,
                                           float stride_px, float aw, float ah) {
  return decode_box(sx, sy, sw, sh, x, y, stride_px, aw, ah);
}
__device__ __forceinline__ float4 pass_box(const TtaDecodeParams& p, int l, float sx, float sy, float sw, float sh, int x,
                                           int y, float stride_px, float aw, float ah) {
  return decode_box_descaled(sx, sy, sw, sh, x, y, stride_px, aw, ah, p.scale[l], p.flip[l] != 0, p.flip_w[l]);
}

template <typename T>
__device__ __forceinline__ float row_elem(const uint8_t* row, int e) {
  if constexpr (std::is_same<T, __half>::value)
    return __half2float(reinterpret_cast<const __half*>(row)[e]);
  else
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(row)[e]);
}

// Params = TtaDecodeParams: the multi-pass variant.  Up to 12 level slices (4 bits of level in the pair word instead of 2:
// PairBits), each box descaled (and un-mirrored) before the corner conversion (pass_box), candidate index anchor * nc +
// class in 32 unsigned bits (candidate_index).  With Params = DecodeParams those helpers are the single-pass kernel's
// own expressions and the instance compiles to the same SASS as before the variant existed.
template <typename T, typename Params>
__global__ void __launch_bounds__(kRowWarps * 32)
decode_rows_kernel(const __grid_constant__ Params p, Workspace ws, int blocks_per_image) {
  extern __shared__ __align__(16) uint8_t s_rows_raw[];     // [kRowWarps][kRowPixels][kRowPitch] | list[kRowList] u64 | pairs[kRowWarps][kRowPairs] uint2
  __shared__ int s_count, s_base, s_maxc;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* s_rows = s_rows_raw + static_cast<size_t>(warp) * kRowPixels * kRowPitch;
  uint64_t* s_list = reinterpret_cast<uint64_t*>(s_rows_raw + static_cast<size_t>(kRowWarps) * kRowPixels * kRowPitch);
  uint2* s_pairs = reinterpret_cast<uint2*>(s_list + kRowList) + warp * kRowPairs;
  const int P = p.pix_start[p.n_levels];                       // pixels per image over all levels
  const int img = blockIdx.x / blocks_per_image;
  const int r0 = (blockIdx.x - img * blocks_per_image) * (kRowWarps * kRowPixels) + warp * kRowPixels;
  const int K = p.n_classes + 5;
  if (threadIdx.x == 0) {
    s_count = 0;
    s_maxc = INT_MIN;
  }
  // this lane's pixel
  const int r = r0 + lane;
  const bool valid = r < P;
  int lv = 0, px = 0, py = 0;
  long long off = 0;
  int row_chunks = 0;                                          // 16-byte chunks of this pixel's row
  if (valid) {
#pragma unroll
    for (int i = 1; i < Params::kLevels; ++i)
      if (i < p.n_levels && r >= p.pix_start[i]) lv = i;
    const yb_head_level& L = p.lvl[lv];
    const int rr = r - p.pix_start[lv];
    py = rr / L.W;
    px = rr - py * L.W;
    off = img * L.stride_n + py * L.stride_y + px * L.stride_x;   // elements
    row_chunks = static_cast<int>(L.stride_x >> 3);
  }
  // rows -> shared memory.  Fast path: the warp's 32 pixels are valid, on one level, and their rows are one contiguous
  // 32 x 512-byte run of the NHWC buffer (dense level: next pixel = +stride_x, rows 512 bytes): every lane issues 32
  // 16-byte cp.async at consecutive addresses -- 3 instructions per copy instead of the ~12 of the per-row loop below
  // (three shuffles + level lookup per row; that loop was about half of the kernel's 17 M warp instructions).
  const uint32_t s_base_addr = smem_u32(s_rows);
  const long long off_first = __shfl_sync(0xffffffffu, off, 0), off_last = __shfl_sync(0xffffffffu, off, 31);
  const int lv_first = __shfl_sync(0xffffffffu, lv, 0), lv_last = __shfl_sync(0xffffffffu, lv, 31);
  const bool dense = __all_sync(0xffffffffu, valid) && lv_first == lv_last && row_chunks == kRowMaxBytes / 16 &&
                     off_last == off_first + 31ll * (kRowMaxBytes / 2);
  if (dense) {
    const uint8_t* src = static_cast<const uint8_t*>(p.lvl[lv_first].logits) + off_first * 2 + lane * 16;
#pragma unroll 8
    for (int j = 0; j < kRowPixels; ++j)   // chunk q = 32 j + lane: row j, 16-byte column `lane`
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s_base_addr + j * kRowPitch + lane * 16), "l"(src + j * kRowMaxBytes) : "memory");
  } else
#pragma unroll 8
  for (int j = 0; j < kRowPixels; ++j) {
    const long long off_j = __shfl_sync(0xffffffffu, off, j);
    const int lv_j = __shfl_sync(0xffffffffu, lv, j);
    const int chunks_j = __shfl_sync(0xffffffffu, row_chunks, j);
    if (lane < chunks_j) {
      const uint8_t* src = static_cast<const uint8_t*>(p.lvl[lv_j].logits) + (off_j + lane * 8) * 2;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s_base_addr + j * kRowPitch + lane * 16), "l"(src) : "memory");
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();                                             // rows landed (own warp) and the block counters are initialised
  // objectness of this lane's pixel, all anchors
  const uint8_t* my_row = s_rows + lane * kRowPitch;
  float obj[YB_MAX_ANCHORS];
  uint32_t pass_bits = 0;
#pragma unroll
  for (int a = 0; a < YB_MAX_ANCHORS; ++a) {
    obj[a] = 0.f;
    if (a < p.n_anchors && valid) {
      obj[a] = sigmoidf_ref(row_elem<T>(my_row, a * K + 4));
      if (obj[a] > p.score_thresh) pass_bits |= 1u << a;   // score = cls*obj <= obj
    }
  }
  float lane_maxc = -INFINITY;
  // Class scan.  The (pixel, anchor) pairs that passed objectness are first COMPACTED across the warp (ballot + prefix
  // popcount into a per-warp list), then lane q takes pair q: with ~20 % of the anchors passing, the lane-owns-pixel
  // scan ran every anchor's loop with ~6 of 32 lanes active (ncu: 18.6 active threads per instruction, the kernel
  // issue-bound at 19.4 M warp instructions); compacted, one pass covers what took three.
  // A raw-logit pre-test spares the exact sigmoid for almost every class: sigmoid(x) * obj > thr  <=>  x > logit(thr/obj);
  // the exact expression (the reference's arithmetic) decides for the few that clear it.  The 1e-2 logit margin dwarfs
  // any rounding; for r -> 1 (obj barely above thr) every x > 15 is tested exactly.
  const uint32_t lt_lanes = (1u << lane) - 1u;
  int n_pairs = 0;
#pragma unroll
  for (int a = 0; a < YB_MAX_ANCHORS; ++a) {
    if (a >= p.n_anchors) break;
    const bool pass = (pass_bits >> a) & 1u;
    const uint32_t bal = __ballot_sync(0xffffffffu, pass);
    if (pass)   // px, py: 10 bits each (maps up to 1023 wide), level, anchor 2, source lane 5
      s_pairs[n_pairs + __popc(bal & lt_lanes)] =
          make_uint2(static_cast<uint32_t>(px) | static_cast<uint32_t>(py) << 10 | static_cast<uint32_t>(lv) << PairBits<Params>::kLv |
                         static_cast<uint32_t>(a) << PairBits<Params>::kAnchor | static_cast<uint32_t>(lane) << PairBits<Params>::kLane,
                     __float_as_uint(obj[a]));
    n_pairs += __popc(bal);
  }
  __syncwarp();
  for (int q = lane; q < n_pairs; q += 32) {
    const uint2 ent = s_pairs[q];
    const int qx = ent.x & 1023, qy = (ent.x >> 10) & 1023, ql = (ent.x >> PairBits<Params>::kLv) & PairBits<Params>::kLvMask,
              a = (ent.x >> PairBits<Params>::kAnchor) & 3;
    const uint8_t* q_row = s_rows + ((ent.x >> PairBits<Params>::kLane) & 31) * kRowPitch;
    const float q_obj = __uint_as_float(ent.y);
    const yb_head_level& L = p.lvl[ql];
    float lt = -INFINITY;
    if (p.score_thresh > 0.f) {
      const float rr = p.score_thresh / q_obj;                 // < 1: the anchor passed obj > thr
      lt = fminf(__logf(rr / (1.0f - rr)) - 1e-2f, 15.0f);
    }
    const int anchor = p.lvl_start[ql] + (a * L.H + qy) * L.W + qx;
    // The class logits of this anchor are elements [e0, e1) of the row; they are walked in aligned 16-byte chunks
    // (8 logits per LDS.128) and pre-tested two at a time in half2 / bfloat162 arithmetic against the threshold
    // rounded DOWN.
    const int e0 = a * K + 5, e1 = a * K + K;
    using T2 = typename std::conditional<std::is_same<T, __half>::value, __half2, __nv_bfloat162>::type;
    T2 lt2;
    if constexpr (std::is_same<T, __half>::value)
      lt2 = __half2half2(__float2half_rd(lt));               // -inf stays -inf: every finite logit clears it
    else
      lt2 = __bfloat162bfloat162(__float2bfloat16_rd(lt));
    bool any = false;
    for (int c = e0 >> 3; c <= (e1 - 1) >> 3; ++c) {
      const uint4 qv = *reinterpret_cast<const uint4*>(q_row + c * 16);
      const uint32_t w[4] = {qv.x, qv.y, qv.z, qv.w};
      uint32_t hit = 0;                                        // bit j: element 8c + j cleared the pre-test
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const T2 v = *reinterpret_cast<const T2*>(&w[j]);
        const T2 g = __hgt2(v, lt2);                           // 1.0 / 0.0 per half
        const uint32_t gb = *reinterpret_cast<const uint32_t*>(&g);
        hit |= ((gb & 0xffffu) ? 1u : 0u) << (2 * j) | ((gb >> 16) ? 1u : 0u) << (2 * j + 1);
      }
      // elements of this chunk that belong to other fields / anchors
      const int lo = e0 - 8 * c, hi = e1 - 8 * c;
      if (lo > 0) hit &= ~((1u << lo) - 1u);
      if (hi < 8) hit &= (1u << hi) - 1u;
      while (hit) {
        const int j = __ffs(hit) - 1;
        hit &= hit - 1;
        const int k = 8 * c + j - e0;
        const float x = row_elem<T>(q_row, 8 * c + j);
        const float score = __fmul_rn(sigmoidf_ref(x), q_obj);
        if (score > p.score_thresh) {
          any = true;
          const uint64_t key = (static_cast<uint64_t>(orderable_desc(score)) << 32) | candidate_index(p, anchor, k);
          const int slot = atomicAdd(&s_count, 1);             // shared-memory atomic: block-local slot
          if (slot < kRowList) {
            s_list[slot] = key;
          } else {   // list full (very low thresholds): straight to the arena
            const int g2 = atomicAdd(&ws.img_count[img], 1);
            if (g2 < p.cap_per_image) ws.keys_a[static_cast<long long>(img) * p.cap_per_image + g2] = key;
          }
        }
      }
    }
    if (any) {
      const float4 b = pass_box(p, ql, sigmoidf_ref(row_elem<T>(q_row, a * K + 0)), sigmoidf_ref(row_elem<T>(q_row, a * K + 1)),
                                sigmoidf_ref(row_elem<T>(q_row, a * K + 2)), sigmoidf_ref(row_elem<T>(q_row, a * K + 3)),
                                qx, qy, L.stride_px, L.anchors_px[2 * a], L.anchors_px[2 * a + 1]);
      ws.boxes[static_cast<long long>(img) * p.anchors_per_image + anchor] = b;
      lane_maxc = fmaxf(lane_maxc, fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w)));
    }
  }
  float warp_maxc = lane_maxc;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) warp_maxc = fmaxf(warp_maxc, __shfl_xor_sync(0xffffffffu, warp_maxc, o));
  if (lane == 0 && warp_maxc > -INFINITY) atomicMax(&s_maxc, float_to_ordered_int(warp_maxc));
  __syncthreads();
  const int n_list = min(s_count, kRowList);
  if (threadIdx.x == 0) {
    s_base = n_list > 0 ? atomicAdd(&ws.img_count[img], n_list) : 0;   // ONE global atomic per block
    if (s_maxc != INT_MIN) atomicMax(&ws.img_maxc[img], s_maxc);
  }
  __syncthreads();
  const int gbase = s_base;
  for (int i = threadIdx.x; i < n_list; i += kRowWarps * 32)
    if (gbase + i < p.cap_per_image) ws.keys_a[static_cast<long long>(img) * p.cap_per_image + gbase + i] = s_list[i];
}

// Dense decode without threshold / NMS (yolort/relay/logits_decoder.py:10-61 = _concat_pred_logits +
// _decode_pred_logits of box_head.py:328-360 for every anchor): one warp per anchor, lane k <-> output k, so the
// (nc+5) logits are read and the nc scores written as contiguous runs. HBM-bound: 2(nc+5) B in, 4(nc+4) B out.
template <typename T>
__global__ void decode_dense_kernel(const __grid_constant__ DecodeParams p, float4* __restrict__ boxes,
                                    float* __restrict__ scores) {
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long total = static_cast<long long>(p.n_images) * p.anchors_per_image;
  if (warp >= total) return;
  const int lane = threadIdx.x & 31;
  const int img = static_cast<int>(warp / p.anchors_per_image);
  const int anchor = static_cast<int>(warp - static_cast<long long>(img) * p.anchors_per_image);
  int l = 0;
#pragma unroll
  for (int i = 1; i < YB_MAX_LEVELS; ++i)
    if (i < p.n_levels && anchor >= p.lvl_start[i]) l = i;
  const yb_head_level& L = p.lvl[l];
  int r = anchor - p.lvl_start[l];
  const int x = r % L.W;
  r /= L.W;
  const int y = r % L.H;
  const int a = r / L.H;
  const long long off = img * L.stride_n + a * L.stride_a + y * L.stride_y + x * L.stride_x;
  const int K = p.n_classes + 5;
  float s0 = 0.f;
  if (lane < K) s0 = sigmoidf_ref(ld_logit<T>(L.logits, off + lane));
  const float sx = __shfl_sync(0xffffffffu, s0, 0), sy = __shfl_sync(0xffffffffu, s0, 1);
  const float sw = __shfl_sync(0xffffffffu, s0, 2), sh = __shfl_sync(0xffffffffu, s0, 3);
  const float obj = __shfl_sync(0xffffffffu, s0, 4);
  if (lane == 0) boxes[warp] = decode_box(sx, sy, sw, sh, x, y, L.stride_px, L.anchors_px[2 * a], L.anchors_px[2 * a + 1]);
  float* out = scores + warp * p.n_classes;
  if (lane >= 5 && lane < K) out[lane - 5] = __fmul_rn(s0, obj);          // box_head.py:357 scores = cls * obj
  for (int k = 32 + lane; k < K; k += 32)
    out[k - 5] = __fmul_rn(sigmoidf_ref(ld_logit<T>(L.logits, off + k)), obj);
}

// ---------------------------------------------------------------------------------------------
// Per-image sort + greedy sweep
// ---------------------------------------------------------------------------------------------
struct NmsParams {
  int n_classes;        // decode mode: label = idx % nc, anchor = idx / nc ; explicit mode: 0
  int anchors_per_image;
  long long cap_per_image;
  float iou_thresh;
  int max_det;
  int semantics;
  int explicit_mode;    // 1: yb_batched_nms (boxes/labels indexed by candidate index)
  const float4* x_boxes;     // explicit mode
  const int64_t* x_labels;   // explicit mode
  const float* rescale;      // [n][3] or null
  float* out_boxes;          // [n][max_det][4]
  float* out_scores;         // [n][max_det]
  int64_t* out_labels;       // [n][max_det]
  int64_t* out_keep;         // explicit mode: [max_det]
  int* out_counts;           // [n]
  long long* status;         // [4]
};

__device__ __forceinline__ float box_area(const float4& b) {
  return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
}
// torchvision/csrc/ops/cpu/nms_kernel.cpp: inter / (iarea + areas[j] - inter) > thr
__device__ __forceinline__ bool iou_over(const float4& a, float area_a, const float4& b, float area_b, float thr) {
  const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
  const float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
  const float w = fmaxf(0.f, __fsub_rn(xx2, xx1));
  const float h = fmaxf(0.f, __fsub_rn(yy2, yy1));
  const float inter = __fmul_rn(w, h);
  // inter == 0 gives ovr = +-0 or NaN (0/0): never "> thr" for thr >= 0, so the IEEE division (a ~40
  // instruction slow path, and the common case: most pairs are disjoint) can be skipped without changing
  // any decision; for thr < 0 fall through to the exact expression.
  if (!(inter > 0.f) && thr >= 0.f) return false;
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
  return ovr > thr;
}

// In-CTA bitonic sort of n (power of two) keys in shared memory.
__device__ void bitonic_sort_smem(uint64_t* keys, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint64_t a = keys[i], b = keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

// Bitonic sort of R * blockDim.x keys (blockDim.x = kNmsThreads) with the keys in REGISTERS: thread t owns elements
// t*R .. t*R+R-1.  Of the log2(n)(log2(n)+1)/2 compare-exchange stages only those whose partner distance reaches into
// another warp (j >= 32 R) go through shared memory with a barrier; distances inside a warp use shuffles and distances
// below R stay inside the thread.  2048 keys: 10 barrier stages instead of 66.  Same network as bitonic_sort_smem, so the same (total) order.
template <int R>
__device__ void bitonic_sort_regs(uint64_t* s) {
  const int tid = threadIdx.x;
  const int n = R * blockDim.x;
  uint64_t v[R];
#pragma unroll
  for (int r = 0; r < R; ++r) v[r] = s[tid * R + r];
  for (int k = 2; k <= n; k <<= 1) {
    int j = k >> 1;
    if (j >= 32 * R) {
      // partners live in other warps: these stages run on the shared-memory copy
      __syncthreads();   // everybody has finished reading the previous contents
#pragma unroll
      for (int r = 0; r < R; ++r) s[tid * R + r] = v[r];
      __syncthreads();
      for (; j >= 32 * R; j >>= 1) {
        for (int pidx = tid; pidx < (n >> 1); pidx += blockDim.x) {
          const int e = ((pidx & ~(j - 1)) << 1) | (pidx & (j - 1));   // element with bit j clear
          const uint64_t a = s[e], b = s[e | j];
          const bool up = (e & k) == 0;
          if ((a > b) == up) {
            s[e] = b;
            s[e | j] = a;
          }
        }
        __syncthreads();
      }
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = s[tid * R + r];
    }
    for (; j >= R; j >>= 1) {          // partner thread in the same warp
      const int m = j / R;
      const bool lower = (tid & m) == 0;
      const bool up = ((tid * R) & k) == 0;
      const bool keep_min = lower == up;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const uint64_t o = __shfl_xor_sync(0xffffffffu, v[r], m);
        // one 64-bit compare and a predicate XOR (a ternary over two compares compiled to divergent branches: 40 % of
        // the kernel's warp samples sat in this loop); equal keys (the ~0 padding) may swap, which changes nothing
        const bool take = (o < v[r]) == keep_min;
        v[r] = take ? o : v[r];
      }
    }
#pragma unroll
    for (int jj = R >> 1; jj >= 1; jj >>= 1) {   // partner register in the same thread (compile-time distances)
      if (2 * jj <= k) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          if ((r & jj) == 0) {
            const bool up = ((tid * R + r) & k) == 0;
            const uint64_t a = v[r], b = v[r | jj];
            const bool sw = (a > b) == up;
            v[r] = sw ? b : a;
            v[r | jj] = sw ? a : b;
          }
        }
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < R; ++r) s[tid * R + r] = v[r];
  __syncthreads();
}

// In-CTA stable LSD radix sort (8-bit digits) of `count` keys living in global memory.
// scratch: hist[256] + base[256] + warp_cnt[32][256] (uint32).  Returns the buffer holding the result.
__device__ uint64_t* block_radix_sort(uint64_t* a, uint64_t* b, int count, uint32_t* scratch) {
  uint32_t* hist = scratch;
  uint32_t* base = scratch + 256;
  uint32_t* wcnt = scratch + 512;  // [32][256]
  __shared__ int s_skip;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t lt_mask = (1u << lane) - 1u;
  const int nwarps = blockDim.x >> 5;
  for (int i = tid; i < nwarps * 256; i += blockDim.x) wcnt[i] = 0;
  for (int pass = 0; pass < 8; ++pass) {
    const int shift = pass * 8;
    if (tid < 256) hist[tid] = 0;
    if (tid == 0) s_skip = 0;
    __syncthreads();
    for (int i = tid; i < count; i += blockDim.x) atomicAdd(&hist[(a[i] >> shift) & 255u], 1u);
    __syncthreads();
    if (tid < 256 && hist[tid] == static_cast<uint32_t>(count)) s_skip = 1;  // digit constant: no-op pass
    __syncthreads();
    if (s_skip) {
      __syncthreads();
      continue;
    }
    if (tid < 32) {  // exclusive scan of 256 bins by one warp, 8 bins per lane
      uint32_t v[8], sum = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[i] = hist[tid * 8 + i];
        sum += v[i];
      }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      uint32_t run = incl - sum;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        base[tid * 8 + i] = run;
        run += v[i];
      }
    }
    __syncthreads();
    for (int t0 = 0; t0 < count; t0 += blockDim.x) {
      const int i = t0 + tid;
      const bool valid = i < count;
      const uint64_t key = valid ? a[i] : 0ull;
      const uint32_t d = valid ? static_cast<uint32_t>((key >> shift) & 255u) : (256u + lane);
      const uint32_t peers = __match_any_sync(0xffffffffu, d);
      const uint32_t rank = __popc(peers & lt_mask);
      const bool leader = valid && rank == 0;
      if (leader) wcnt[warp * 256 + d] = __popc(peers);
      __syncthreads();
      if (tid < 256) {  // per-digit exclusive scan across the warps, continuing the running base
        uint32_t run = base[tid];
        for (int w = 0; w < nwarps; ++w) {
          const uint32_t t = wcnt[w * 256 + tid];
          wcnt[w * 256 + tid] = run;
          run += t;
        }
        base[tid] = run;
      }
      __syncthreads();
      if (valid) b[wcnt[warp * 256 + d] + rank] = key;
      __syncthreads();
      if (tid < 256) {
        for (int w = 0; w < nwarps; ++w) wcnt[w * 256 + tid] = 0;
      }
      __syncthreads();
    }
    uint64_t* t = a;
    a = b;
    b = t;
    __syncthreads();
  }
  return a;
}

// Greedy sweep of one image.  Candidates (already sorted) are consumed kSweep at a time:
//   A. every thread tests its candidate against the kept list (<= max_det boxes, shared memory);
//   B. survivors are compacted in order and their pairwise suppression bit-matrix is built in parallel;
//   C. warp 0 walks the survivors in order with the bit-matrix (one 32-bit word of the "removed" set per
//      lane, warp shuffles only) -- the sequential part costs ~20 cycles per survivor;
//   D. kept survivors are appended to the kept list / written out in parallel.
__global__ void __launch_bounds__(kNmsThreads)
nms_image_kernel(const NmsParams p, Workspace ws) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  // layout: [sort region 36 KB: 4096 keys | radix scratch] [survivors] [bit matrix] [kept list]
  uint64_t* s_keys = reinterpret_cast<uint64_t*>(dyn_smem);
  uint32_t* s_scratch = reinterpret_cast<uint32_t*>(dyn_smem);
  float4* sv_box = reinterpret_cast<float4*>(dyn_smem + 36 * 1024);          // [kSweep] (offset) boxes
  float4* sv_obox = sv_box + kSweep;                                          // [kSweep] original boxes
  float* sv_area = reinterpret_cast<float*>(sv_obox + kSweep);                // [kSweep]
  float* sv_score = sv_area + kSweep;                                         // [kSweep]
  int* sv_label = reinterpret_cast<int*>(sv_score + kSweep);                  // [kSweep]
  uint32_t* sv_cidx = reinterpret_cast<uint32_t*>(sv_label + kSweep);         // [kSweep]
  uint32_t* s_mask = sv_cidx + kSweep;                                        // [kSweep][kSweep/32]
  uint32_t* s_labmask = s_mask + kSweep * (kSweep / 32);                      // [kMaxLabelMasks][kSweep/32]
  float4* k_box = reinterpret_cast<float4*>(s_labmask + kMaxLabelMasks * (kSweep / 32)); // [max_det]
  float* k_area = reinterpret_cast<float*>(k_box + p.max_det);
  int* k_label = reinterpret_cast<int*>(k_area + p.max_det);
  __shared__ int s_kcount, s_warp_tot[kNmsThreads / 32], s_nsurv, s_newkept;
  __shared__ uint32_t s_keep[kSweep / 32];

  const int img = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  long long t_prev = clock64();
  int t_slot = 4;
#define YB_NMS_TICK()                                            \
  do {                                                           \
    if (img == 0 && tid == 0 && t_slot < 16) {                   \
      const long long t_now = clock64();                         \
      ws.status[t_slot++] += t_now - t_prev;                     \
      t_prev = t_now;                                            \
    }                                                            \
  } while (0)
  const long long raw_count = ws.img_count[img];
  const int count = static_cast<int>(raw_count < p.cap_per_image ? raw_count : p.cap_per_image);
  if (tid == 0) {
    atomicAdd(reinterpret_cast<unsigned long long*>(&p.status[0]), static_cast<unsigned long long>(raw_count));
    atomicMax(reinterpret_cast<unsigned long long*>(&p.status[2]), static_cast<unsigned long long>(raw_count));
    if (raw_count > p.cap_per_image) {
      atomicExch(reinterpret_cast<unsigned long long*>(&p.status[1]), 1ull);
      p.out_counts[img] = 0;
    }
    s_kcount = 0;
  }
  if (raw_count > p.cap_per_image) return;  // host grows the arena and re-runs

  uint64_t* keys_g = ws.keys_a + static_cast<long long>(img) * p.cap_per_image;
  const uint64_t* sorted;
  if (count <= kSmallSort) {
    // padded to 4 (8) keys per thread with keys that sort last
    const int n2 = count <= 4 * kNmsThreads ? 4 * kNmsThreads : 8 * kNmsThreads;
    for (int i = tid; i < n2; i += blockDim.x) s_keys[i] = i < count ? keys_g[i] : ~0ull;
    __syncthreads();
    if (n2 == 4 * kNmsThreads)
      bitonic_sort_regs<4>(s_keys);
    else
      bitonic_sort_regs<8>(s_keys);
    sorted = s_keys;
  } else {
    __syncthreads();
    sorted = block_radix_sort(keys_g, ws.keys_b + static_cast<long long>(img) * p.cap_per_image, count, s_scratch);
  }
  __syncthreads();
  YB_NMS_TICK();  // slot 4: load + sort

  bool trick;
  if (p.semantics == YB_NMS_TV_AUTO)
    trick = static_cast<long long>(count) * 4 <= 4000;  // torchvision: boxes.numel() > 4000 -> per-class
  else
    trick = p.semantics == YB_NMS_OFFSET_TRICK;
  float off_unit = 0.f;
  if (trick) off_unit = __fadd_rn(ordered_int_to_float(ws.img_maxc[img]), 1.0f);  // max_coordinate + 1

  float gain = 1.f, padx = 0.f, pady = 0.f;
  if (p.rescale) {
    gain = p.rescale[img * 3 + 0];
    padx = p.rescale[img * 3 + 1];
    pady = p.rescale[img * 3 + 2];
  }
  const uint32_t lt_mask = (1u << lane) - 1u;

  for (int base = 0; base < count; base += kSweep) {
    // ---- A: fetch + test against the kept list ----
    const int j = base + tid;
    bool alive = j < count;
    float4 box = make_float4(0.f, 0.f, 0.f, 0.f), nbox = box;
    float area = 0.f, score = 0.f;
    int label = 0;
    uint32_t cidx = 0;
    if (alive) {
      const uint64_t key = sorted[j];
      score = from_orderable_desc(static_cast<uint32_t>(key >> 32));
      cidx = static_cast<uint32_t>(key);
      if (p.explicit_mode) {
        box = p.x_boxes[cidx];
        label = static_cast<int>(p.x_labels[cidx]);
      } else {
        const int anchor = cidx / p.n_classes;
        label = cidx - anchor * p.n_classes;
        box = ws.boxes[static_cast<long long>(img) * p.anchors_per_image + anchor];
      }
      nbox = box;
      if (trick) {
        const float off = __fmul_rn(static_cast<float>(label), off_unit);
        nbox = make_float4(__fadd_rn(box.x, off), __fadd_rn(box.y, off), __fadd_rn(box.z, off), __fadd_rn(box.w, off));
      }
      area = box_area(nbox);
      const int kc = s_kcount;
      bool hit = false;
#pragma unroll 4
      for (int i = 0; i < kc; ++i) {   // no early exit: independent iterations pipeline their loads
        const bool same = trick || k_label[i] == label;
        hit |= same && iou_over(k_box[i], k_area[i], nbox, area, p.iou_thresh);
      }
      alive = !hit;
    }
    if (base == 0) YB_NMS_TICK();  // slot 5: phase A (first batch)
    // ---- B: order-preserving compaction of the survivors ----
    const uint32_t bal = __ballot_sync(0xffffffffu, alive);
    if (lane == 0) s_warp_tot[warp] = __popc(bal);
    __syncthreads();
    int pos = __popc(bal & lt_mask);
    for (int w = 0; w < warp; ++w) pos += s_warp_tot[w];
    if (tid == 0) {
      int t = 0;
      for (int w = 0; w < kNmsThreads / 32; ++w) t += s_warp_tot[w];
      s_nsurv = t;
    }
    if (alive) {
      sv_box[pos] = nbox;
      sv_obox[pos] = box;
      sv_area[pos] = area;
      sv_score[pos] = score;
      sv_label[pos] = label;
      sv_cidx[pos] = cidx;
    }
    if (tid < kSweep / 32) s_keep[tid] = 0;
    const bool use_labmask = !trick && !p.explicit_mode && p.n_classes <= kMaxLabelMasks;
    if (use_labmask)
      for (int i = tid; i < p.n_classes * (kSweep / 32); i += blockDim.x) s_labmask[i] = 0;
    __syncthreads();
    const int S = s_nsurv;
    const int nwords = (S + 31) >> 5;
    if (use_labmask) {   // bit i of s_labmask[word][label] <=> survivor i carries that label (label-minor: lanes with
                         // different labels hit different banks)
      if (tid < S) atomicOr(&s_labmask[(tid >> 5) * p.n_classes + sv_label[tid]], 1u << (tid & 31));
      __syncthreads();
    }
    if (base == 0) YB_NMS_TICK();  // slot 6: compaction
    // suppression bit-matrix: bit j of row i set iff survivor i (if kept) suppresses survivor j > i.  Only the words
    // w >= i / 32 of a row are ever read; those (row, word) pairs are enumerated word-major (word w has
    // min(S, 32 (w + 1)) rows) and dealt out round-robin, so every thread gets the same number of pairs -- with one
    // thread per ROW the first warp walked 16 words per thread while the last walked one (70 k of the kernel's 185 k
    // cycles were this triangle's critical path).
    {
      int w = 0, acc = 0;                         // pairs [acc, acc + rows(w)) belong to word w
      for (int q = tid;; q += blockDim.x) {
        while (w < nwords && q >= acc + min(S, 32 * (w + 1))) {
          acc += min(S, 32 * (w + 1));
          ++w;
        }
        if (w >= nwords) break;
        const int i = q - acc;
        const float4 bi = sv_box[i];
        const float ai = sv_area[i];
        const int li = sv_label[i];
        uint32_t bits = 0;
        const int j0 = w << 5;
        if (j0 + 31 > i) {
          // step 1: which later survivors can this one suppress at all (same class, or any in offset-trick mode)
          uint32_t cand;
          const int jend = min(32, S - j0);
          if (trick) {
            cand = jend == 32 ? 0xffffffffu : ((1u << jend) - 1u);
          } else if (use_labmask) {
            cand = s_labmask[w * p.n_classes + li];
          } else {
            cand = 0;
            for (int b = 0; b < jend; ++b) cand |= (sv_label[j0 + b] == li ? 1u : 0u) << b;
          }
          if (j0 <= i) cand &= ~((2u << (i - j0)) - 1u);   // only j > i
          // step 2: IoU only for those, two per iteration (independent chains: the loads and the division overlap)
          while (cand) {
            const int b0 = __ffs(cand) - 1;
            cand &= cand - 1;
            const bool two = cand != 0;
            const int b1 = two ? __ffs(cand) - 1 : b0;
            cand &= cand - 1;          // no-op when cand is already 0
            const bool o0 = iou_over(bi, ai, sv_box[j0 + b0], sv_area[j0 + b0], p.iou_thresh);
            const bool o1 = iou_over(bi, ai, sv_box[j0 + b1], sv_area[j0 + b1], p.iou_thresh);
            bits |= (o0 ? 1u : 0u) << b0;
            bits |= (o1 ? 1u : 0u) << b1;   // b1 == b0 when there was only one: same bit
          }
        }
        s_mask[i * (kSweep / 32) + w] = bits;
      }
    }
    __syncthreads();
    if (base == 0) YB_NMS_TICK();  // slot 7: bit-matrix (includes the barrier before)
    // ---- C: sequential resolution ----
    // One thread walks the survivors in order; the "removed" set (<= 512 bits) lives in 16 registers, so the
    // only memory traffic is 16 independent shared-memory loads per KEPT survivor (no cross-lane exchange on
    // the critical path).
    if (warp == 0) {
      // Survivors are resolved 32 at a time.  Inside a chunk the decision chain runs on registers only: every lane holds
      // the chunk's 32 x 32 diagonal block (32 broadcast loads, issued up front) and walks the 32 survivors with a
      // 4-instruction dependent chain each; the rows of the survivors that were kept are then OR-ed into the removed
      // words of the LATER chunks by the lanes that own them (independent loads).  The one-survivor-at-a-time loop cost
      // ~90 cycles per survivor (a shared-memory load and a vote on the critical path): 45 k of the kernel's 185 k cycles.
      uint32_t removed = 0, keep = 0;   // lane l owns word l of both sets (S <= 512 -> 16 words)
      int kc = s_kcount;
      const int kc0 = kc;
      for (int c = 0; c < nwords && kc < p.max_det; ++c) {
        uint32_t diag[32];
#pragma unroll
        for (int b = 0; b < 32; ++b) diag[b] = (32 * c + b < S) ? s_mask[(32 * c + b) * (kSweep / 32) + c] : 0xffffffffu;
        uint32_t rem_c = __shfl_sync(0xffffffffu, removed, c);
        if (S - 32 * c < 32) rem_c |= ~((1u << (S - 32 * c)) - 1u);   // positions past the last survivor
        uint32_t keep_c = 0;
#pragma unroll
        for (int b = 0; b < 32; ++b) {
          const bool take = !((rem_c >> b) & 1u) && kc < p.max_det;
          kc += take ? 1 : 0;
          keep_c |= (take ? 1u : 0u) << b;
          rem_c |= take ? diag[b] : 0u;
        }
        if (lane == c) keep = keep_c;
        if (lane > c && lane < nwords) {   // 32 predicated, independent loads (a data-dependent loop would serialise their latency)
#pragma unroll
          for (int b = 0; b < 32; ++b)
            if ((keep_c >> b) & 1u) removed |= s_mask[(32 * c + b) * (kSweep / 32) + lane];
        }
      }
      if (lane < kSweep / 32) s_keep[lane] = keep;
      if (lane == 0) s_newkept = kc - kc0;
    }
    __syncthreads();
    if (base == 0) YB_NMS_TICK();  // slot 8: resolve
    // ---- D: append the kept survivors ----
    if (tid < S && ((s_keep[tid >> 5] >> (tid & 31)) & 1u)) {
      int rank = __popc(s_keep[tid >> 5] & ((1u << (tid & 31)) - 1u));
      for (int w = 0; w < (tid >> 5); ++w) rank += __popc(s_keep[w]);
      const int slot = s_kcount + rank;
      k_box[slot] = sv_box[tid];
      k_area[slot] = sv_area[tid];
      k_label[slot] = sv_label[tid];
      const long long o = static_cast<long long>(img) * p.max_det + slot;
      if (p.explicit_mode) {
        p.out_keep[slot] = static_cast<int64_t>(sv_cidx[tid]);
      } else {
        float4 ob = sv_obox[tid];
        if (p.rescale) {  // transform.py:362-365: (x - pad) / gain, fp32, no clipping
          ob.x = __fdiv_rn(__fsub_rn(ob.x, padx), gain);
          ob.z = __fdiv_rn(__fsub_rn(ob.z, padx), gain);
          ob.y = __fdiv_rn(__fsub_rn(ob.y, pady), gain);
          ob.w = __fdiv_rn(__fsub_rn(ob.w, pady), gain);
        }
        reinterpret_cast<float4*>(p.out_boxes)[o] = ob;
        p.out_scores[o] = sv_score[tid];
        p.out_labels[o] = static_cast<int64_t>(sv_label[tid]);
      }
    }
    __syncthreads();
    if (tid == 0) s_kcount += s_newkept;
    __syncthreads();
    if (s_kcount >= p.max_det) break;
  }
  __syncthreads();
  YB_NMS_TICK();  // slot 9: append + remaining batches
  if (tid == 0) p.out_counts[img] = s_kcount;
#undef YB_NMS_TICK
}

// explicit-candidate key builder for yb_batched_nms
__global__ void build_keys_kernel(const float* __restrict__ scores, const float4* __restrict__ boxes,
                                  long long n, Workspace ws) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ws.keys_a[i] = (static_cast<uint64_t>(orderable_desc(scores[i])) << 32) | static_cast<uint32_t>(i);
  const float4 b = boxes[i];
  atomicMax(&ws.img_maxc[0], float_to_ordered_int(fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w))));
}

__global__ void init_counters_kernel(Workspace ws, int n, long long* status, int preset_count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    ws.img_count[i] = preset_count;
    ws.img_maxc[i] = float_to_ordered_int(-INFINITY);
  }
  if (i < 4 && status) status[i] = 0;
  if (i < 16) ws.status[i] = 0;
}

size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

size_t carve(Workspace& ws, uint8_t* base, int n, long long cap, long long anchors) {
  size_t off = 0;
  ws.keys_a = reinterpret_cast<uint64_t*>(base + off);
  off += align256(static_cast<size_t>(n) * cap * 8);
  ws.keys_b = reinterpret_cast<uint64_t*>(base + off);
  off += align256(static_cast<size_t>(n) * cap * 8);
  ws.boxes = reinterpret_cast<float4*>(base + off);
  off += align256(static_cast<size_t>(n) * anchors * 16);
  ws.img_count = reinterpret_cast<int*>(base + off);
  off += align256(static_cast<size_t>(n) * 4);
  ws.img_maxc = reinterpret_cast<int*>(base + off);
  off += align256(static_cast<size_t>(n) * 4);
  ws.status = reinterpret_cast<long long*>(base + off);
  off += align256(16 * sizeof(long long));   // [0,4) status, [4,16) phase timers of image 0 (debug)
  return off;
}

size_t nms_smem_bytes(int max_det) {
  return 36 * 1024 + static_cast<size_t>(kSweep) * (16 + 16 + 4 + 4 + 4 + 4) + static_cast<size_t>(kSweep) * (kSweep / 32) * 4 +
         static_cast<size_t>(kMaxLabelMasks) * (kSweep / 32) * 4 + static_cast<size_t>(max_det) * (16 + 4 + 4);
}

int ensure_nms_smem(size_t bytes) {
  static size_t configured = 0;
  if (bytes > configured) {
    YB_CHECK_CUDA(cudaFuncSetAttribute(nms_image_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(bytes)));
    configured = bytes;
  }
  return YB_OK;
}

long long anchors_per_image(const yb_nms_params* p, const yb_head_level* lv) {
  long long a = 0;
  for (int l = 0; l < p->n_levels; ++l) a += static_cast<long long>(p->n_anchors) * lv[l].H * lv[l].W;
  return a;
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" size_t yb_decode_nms_workspace_bytes(const yb_nms_params* p, const yb_head_level* levels) {
  if (!p || !levels || p->n_images <= 0 || p->n_levels <= 0 || p->n_levels > YB_MAX_LEVELS) return 0;
  Workspace ws;
  const long long cap = (p->max_candidates + p->n_images - 1) / p->n_images;
  return carve(ws, nullptr, p->n_images, cap > 0 ? cap : 1, anchors_per_image(p, levels));
}

// debug: byte offset, inside the workspace, of 16 int64 words: [4..10) = per-phase clock counts of image 0
extern "C" size_t yb_decode_nms_debug_offset(const yb_nms_params* p, const yb_head_level* levels) {
  if (!p || !levels || p->n_images <= 0) return 0;
  Workspace ws;
  const long long cap = (p->max_candidates + p->n_images - 1) / p->n_images;
  carve(ws, nullptr, p->n_images, cap > 0 ? cap : 1, anchors_per_image(p, levels));
  return reinterpret_cast<size_t>(ws.status);
}

namespace {
// validates the arguments shared by the entry points below and carves the workspace
int prepare(const yb_nms_params* p, const yb_head_level* levels, void* workspace_dev, size_t workspace_bytes,
            Workspace& ws, long long& apm, long long& cap) {
  YB_REQUIRE(p && levels && workspace_dev, "decode_nms: null argument");
  YB_REQUIRE(p->n_images > 0 && p->n_levels > 0 && p->n_levels <= YB_MAX_LEVELS, "decode_nms: n_images/n_levels");
  YB_REQUIRE(p->n_anchors > 0 && p->n_anchors <= YB_MAX_ANCHORS && p->n_classes > 0, "decode_nms: anchors/classes");
  YB_REQUIRE(p->max_det > 0 && p->max_det <= 4096, "decode_nms: max_det must be in [1, 4096]");
  YB_REQUIRE(p->semantics >= 0 && p->semantics <= 2, "decode_nms: bad semantics");
  apm = anchors_per_image(p, levels);
  YB_REQUIRE(apm > 0, "decode_nms: no anchors");
  YB_REQUIRE(apm * p->n_classes < (1ll << 31), "decode_nms: anchors*classes overflows the candidate index");
  cap = (p->max_candidates + p->n_images - 1) / p->n_images;
  YB_REQUIRE(cap >= 1, "decode_nms: max_candidates too small");
  const size_t need = carve(ws, static_cast<uint8_t*>(workspace_dev), p->n_images, cap, apm);
  if (need > workspace_bytes) {
    set_error("decode_nms: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  return YB_OK;
}
}  // namespace

extern "C" int yb_nms_layout(const yb_nms_params* p, const yb_head_level* levels, void* workspace_dev,
                             size_t workspace_bytes, yb_nms_layout_t* out) {
  YB_REQUIRE(out != nullptr, "nms_layout: null output");
  Workspace ws;
  long long apm, cap;
  int rc = prepare(p, levels, workspace_dev, workspace_bytes, ws, apm, cap);
  if (rc != YB_OK) return rc;
  out->keys = ws.keys_a;
  out->boxes = ws.boxes;
  out->img_count = ws.img_count;
  out->img_maxc = ws.img_maxc;
  out->cap_per_image = cap;
  out->anchors_per_image = static_cast<int32_t>(apm);
  int start = 0;
  for (int l = 0; l < YB_MAX_LEVELS; ++l) {
    out->level_start[l] = start;
    if (l < p->n_levels) start += p->n_anchors * levels[l].H * levels[l].W;
  }
  return YB_OK;
}

extern "C" int yb_nms_begin(const yb_nms_params* p, const yb_head_level* levels, int64_t* status_dev,
                            void* workspace_dev, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(status_dev != nullptr, "nms_begin: null status");
  Workspace ws;
  long long apm, cap;
  int rc = prepare(p, levels, workspace_dev, workspace_bytes, ws, apm, cap);
  if (rc != YB_OK) return rc;
  init_counters_kernel<<<(p->n_images + 127) / 128 + 1, 128, 0, stream>>>(ws, p->n_images,
                                                                          reinterpret_cast<long long*>(status_dev), 0);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

namespace {
// sort + sweep + rescale of the decoded candidates in `ws` (anchors_per_image `apm`, arena share `cap` per image)
int launch_nms(const yb_nms_params* p, long long apm, long long cap, const Workspace& ws, const float* rescale_dev,
               float* boxes_dev, float* scores_dev, int64_t* labels_dev, int32_t* counts_dev, int64_t* status_dev,
               cudaStream_t stream) {
  NmsParams np;
  np.n_classes = p->n_classes;
  np.anchors_per_image = static_cast<int>(apm);
  np.cap_per_image = cap;
  np.iou_thresh = p->iou_thresh;
  np.max_det = p->max_det;
  np.semantics = p->semantics;
  np.explicit_mode = 0;
  np.x_boxes = nullptr;
  np.x_labels = nullptr;
  np.rescale = rescale_dev;
  np.out_boxes = boxes_dev;
  np.out_scores = scores_dev;
  np.out_labels = labels_dev;
  np.out_keep = nullptr;
  np.out_counts = counts_dev;
  np.status = reinterpret_cast<long long*>(status_dev);
  const size_t smem = nms_smem_bytes(p->max_det);
  const int rc = ensure_nms_smem(smem);
  if (rc != YB_OK) return rc;
  nms_image_kernel<<<p->n_images, kNmsThreads, smem, stream>>>(np, ws);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
}  // namespace

extern "C" int yb_nms_finish(const yb_nms_params* p, const yb_head_level* levels, const float* rescale_dev,
                             float* boxes_dev, float* scores_dev, int64_t* labels_dev, int32_t* counts_dev,
                             int64_t* status_dev, void* workspace_dev, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(boxes_dev && scores_dev && labels_dev && counts_dev && status_dev, "nms_finish: null output");
  Workspace ws;
  long long apm, cap;
  int rc = prepare(p, levels, workspace_dev, workspace_bytes, ws, apm, cap);
  if (rc != YB_OK) return rc;
  return launch_nms(p, apm, cap, ws, rescale_dev, boxes_dev, scores_dev, labels_dev, counts_dev, status_dev, stream);
}

namespace yb {
namespace {
int fill_decode_params(const yb_nms_params* p, const yb_head_level* levels, DecodeParams& dp, int& dtype) {
  YB_REQUIRE(p && levels, "decode: null argument");
  YB_REQUIRE(p->n_images > 0 && p->n_levels > 0 && p->n_levels <= YB_MAX_LEVELS, "decode: n_images/n_levels");
  YB_REQUIRE(p->n_anchors > 0 && p->n_anchors <= YB_MAX_ANCHORS && p->n_classes > 0, "decode: n_anchors/n_classes");
  dtype = levels[0].dtype;
  dp.lvl_start[0] = 0;
  for (int l = 0; l < YB_MAX_LEVELS; ++l) {
    if (l < p->n_levels) {
      YB_REQUIRE(levels[l].dtype == dtype, "decode: all levels must share a dtype");
      YB_REQUIRE(levels[l].logits != nullptr && levels[l].H > 0 && levels[l].W > 0, "decode: level %d empty", l);
      dp.lvl[l] = levels[l];
      dp.lvl_start[l + 1] = dp.lvl_start[l] + p->n_anchors * levels[l].H * levels[l].W;
    } else {
      dp.lvl[l] = levels[0];
      dp.lvl_start[l + 1] = dp.lvl_start[l];
    }
  }
  dp.n_images = p->n_images;
  dp.n_levels = p->n_levels;
  dp.n_anchors = p->n_anchors;
  dp.n_classes = p->n_classes;
  dp.anchors_per_image = dp.lvl_start[p->n_levels];
  dp.score_thresh = p->score_thresh;
  dp.cap_per_image = 0;
  return YB_OK;
}
}  // namespace
}  // namespace yb

extern "C" int yb_decode_dense(const yb_nms_params* p, const yb_head_level* levels, float* boxes_dev, float* scores_dev,
                               void* stream_) {
  using namespace yb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(boxes_dev && scores_dev, "decode_dense: null output");
  DecodeParams dp;
  int dtype = 0;
  const int rc = fill_decode_params(p, levels, dp, dtype);
  if (rc != YB_OK) return rc;
  const long long total = static_cast<long long>(dp.n_images) * dp.anchors_per_image;
  YB_REQUIRE(total * 32 / 256 + 1 < (1ll << 31), "decode_dense: too many anchors");
  const unsigned blocks = static_cast<unsigned>((total * 32 + 255) / 256);
  float4* b4 = reinterpret_cast<float4*>(boxes_dev);
  switch (dtype) {
    case YB_F32:
      decode_dense_kernel<float><<<blocks, 256, 0, stream>>>(dp, b4, scores_dev);
      break;
    case YB_F16:
      decode_dense_kernel<__half><<<blocks, 256, 0, stream>>>(dp, b4, scores_dev);
      break;
    case YB_BF16:
      decode_dense_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(dp, b4, scores_dev);
      break;
    default:
      set_error("decode_dense: unsupported logits dtype %d", dtype);
      return YB_ERR_INVALID;
  }
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_decode_candidates(const yb_nms_params* p, const yb_head_level* levels, void* workspace_dev,
                                    size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Workspace ws;
  long long apm, cap;
  int rc = prepare(p, levels, workspace_dev, workspace_bytes, ws, apm, cap);
  if (rc != YB_OK) return rc;
  DecodeParams dp;
  const int dtype = levels[0].dtype;
  dp.lvl_start[0] = 0;
  for (int l = 0; l < YB_MAX_LEVELS; ++l) {
    if (l < p->n_levels) {
      YB_REQUIRE(levels[l].dtype == dtype, "decode_nms: all levels must share a dtype");
      YB_REQUIRE(levels[l].logits != nullptr && levels[l].H > 0 && levels[l].W > 0, "decode_nms: level %d empty", l);
      dp.lvl[l] = levels[l];
      dp.lvl_start[l + 1] = dp.lvl_start[l] + p->n_anchors * levels[l].H * levels[l].W;
    } else {
      dp.lvl[l] = levels[0];
      dp.lvl_start[l + 1] = dp.lvl_start[l];
    }
  }
  dp.n_images = p->n_images;
  dp.n_levels = p->n_levels;
  dp.n_anchors = p->n_anchors;
  dp.n_classes = p->n_classes;
  dp.anchors_per_image = static_cast<int>(apm);
  dp.score_thresh = p->score_thresh;
  dp.cap_per_image = cap;
  // NHWC rows (the plan's head buffers): every level is [.., A*K logits of one pixel, pad] with 16-bit elements,
  // a 16-byte aligned pitch of at most 512 bytes -> the coalesced row kernel; anything else (the reference's
  // [N,A,H,W,K] layout, fp32 logits) -> one thread per anchor.
  bool rows = (dtype == YB_F16 || dtype == YB_BF16) && p->n_anchors <= YB_MAX_ANCHORS;
  dp.pix_start[0] = 0;
  for (int l = 0; l < YB_MAX_LEVELS; ++l) {
    const bool on = l < p->n_levels;
    dp.pix_start[l + 1] = dp.pix_start[l] + (on ? levels[l].H * levels[l].W : 0);
    if (on) {
      const yb_head_level& L = levels[l];
      rows = rows && L.stride_a == p->n_classes + 5 && L.stride_x % 8 == 0 && L.stride_x * 2 <= kRowMaxBytes &&
             L.stride_x >= static_cast<long long>(p->n_anchors) * (p->n_classes + 5) && L.stride_y % 8 == 0 && L.stride_n % 8 == 0 &&
             (reinterpret_cast<uintptr_t>(L.logits) & 15) == 0;
    }
  }
  const long long total = static_cast<long long>(p->n_images) * apm;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  if (rows) {
    const int bpi = (dp.pix_start[p->n_levels] + kRowWarps * kRowPixels - 1) / (kRowWarps * kRowPixels);   // blocks per image
    const unsigned rblocks = static_cast<unsigned>(p->n_images) * static_cast<unsigned>(bpi);
    constexpr int kRowSmem = kRowWarps * kRowPixels * kRowPitch + kRowList * 8 + kRowWarps * kRowPairs * 8;   // 66 KB rows + 4 KB candidate list + 4 KB pair lists
    static bool configured = false;
    if (!configured) {
      YB_CHECK_CUDA(cudaFuncSetAttribute(decode_rows_kernel<__half, DecodeParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRowSmem));
      YB_CHECK_CUDA(cudaFuncSetAttribute(decode_rows_kernel<__nv_bfloat16, DecodeParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRowSmem));
      configured = true;
    }
    if (dtype == YB_F16)
      decode_rows_kernel<__half, DecodeParams><<<rblocks, kRowWarps * 32, kRowSmem, stream>>>(dp, ws, bpi);
    else
      decode_rows_kernel<__nv_bfloat16, DecodeParams><<<rblocks, kRowWarps * 32, kRowSmem, stream>>>(dp, ws, bpi);
    YB_CHECK_CUDA(cudaGetLastError());
    return YB_OK;
  }
  switch (dtype) {
    case YB_F32:
      decode_candidates_kernel<float><<<blocks, 256, 0, stream>>>(dp, ws);
      break;
    case YB_F16:
      decode_candidates_kernel<__half><<<blocks, 256, 0, stream>>>(dp, ws);
      break;
    case YB_BF16:
      decode_candidates_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(dp, ws);
      break;
    default:
      set_error("decode_nms: unsupported logits dtype %d", dtype);
      return YB_ERR_INVALID;
  }
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" int yb_decode_nms(const yb_nms_params* p, const yb_head_level* levels, const float* rescale_dev,
                             float* boxes_dev, float* scores_dev, int64_t* labels_dev, int32_t* counts_dev,
                             int64_t* status_dev, void* workspace_dev, size_t workspace_bytes, void* stream_) {
  int rc = yb_nms_begin(p, levels, status_dev, workspace_dev, workspace_bytes, stream_);
  if (rc != YB_OK) return rc;
  rc = yb_decode_candidates(p, levels, workspace_dev, workspace_bytes, stream_);
  if (rc != YB_OK) return rc;
  return yb_nms_finish(p, levels, rescale_dev, boxes_dev, scores_dev, labels_dev, counts_dev, status_dev, workspace_dev,
                       workspace_bytes, stream_);
}

extern "C" size_t yb_batched_nms_workspace_bytes(int64_t n_boxes) {
  Workspace ws;
  return carve(ws, nullptr, 1, n_boxes > 0 ? n_boxes : 1, 1);
}

extern "C" int yb_batched_nms(const float* boxes_dev, const float* scores_dev, const int64_t* labels_dev,
                              int64_t n_boxes, float iou_thresh, int semantics, int32_t max_keep,
                              int64_t* keep_dev, int32_t* n_keep_dev, void* workspace_dev,
                              size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(keep_dev && n_keep_dev && workspace_dev, "batched_nms: null argument");
  YB_REQUIRE(n_boxes >= 0 && n_boxes < (1ll << 31), "batched_nms: n_boxes out of range");
  YB_REQUIRE(max_keep > 0 && max_keep <= 4096, "batched_nms: max_keep must be in [1, 4096]");
  YB_REQUIRE(semantics >= 0 && semantics <= 2, "batched_nms: bad semantics");
  YB_REQUIRE(n_boxes == 0 || (boxes_dev && scores_dev && labels_dev), "batched_nms: null inputs");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(boxes_dev) & 15) == 0, "batched_nms: boxes must be 16-byte aligned");
  Workspace ws;
  const long long cap = n_boxes > 0 ? n_boxes : 1;
  const size_t need = carve(ws, static_cast<uint8_t*>(workspace_dev), 1, cap, 1);
  if (need > workspace_bytes) {
    set_error("batched_nms: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  init_counters_kernel<<<1, 128, 0, stream>>>(ws, 1, ws.status, static_cast<int>(n_boxes));
  YB_CHECK_CUDA(cudaGetLastError());
  if (n_boxes > 0) {
    build_keys_kernel<<<static_cast<unsigned>((n_boxes + 255) / 256), 256, 0, stream>>>(
        scores_dev, reinterpret_cast<const float4*>(boxes_dev), n_boxes, ws);
    YB_CHECK_CUDA(cudaGetLastError());
  }
  NmsParams np;
  np.n_classes = 0;
  np.anchors_per_image = 0;
  np.cap_per_image = cap;
  np.iou_thresh = iou_thresh;
  np.max_det = max_keep;
  np.semantics = semantics;
  np.explicit_mode = 1;
  np.x_boxes = reinterpret_cast<const float4*>(boxes_dev);
  np.x_labels = labels_dev;
  np.rescale = nullptr;
  np.out_boxes = nullptr;
  np.out_scores = nullptr;
  np.out_labels = nullptr;
  np.out_keep = keep_dev;
  np.out_counts = n_keep_dev;
  np.status = ws.status;  // not reported through this entry point
  const size_t smem = nms_smem_bytes(max_keep);
  int rc = ensure_nms_smem(smem);
  if (rc != YB_OK) return rc;
  nms_image_kernel<<<1, kNmsThreads, smem, stream>>>(np, ws);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

// ---------------------------------------------------------------------------------------------
// Test-time augmentation: one per-image candidate arena over every pass (v5/models/yolo.py:152-163)
// ---------------------------------------------------------------------------------------------
namespace {
// validates the passes and fills the multi-pass decode parameters; `apm` = kept anchors per image over all passes
int fill_tta_params(const yb_nms_params* p, int n_passes, const yb_tta_pass* passes, TtaDecodeParams& dp, int& dtype,
                    long long& apm) {
  YB_REQUIRE(p && passes, "decode_nms_tta: null argument");
  YB_REQUIRE(p->n_images > 0, "decode_nms_tta: n_images");
  YB_REQUIRE(n_passes > 0 && n_passes <= YB_TTA_MAX_PASSES, "decode_nms_tta: 1..%d passes", YB_TTA_MAX_PASSES);
  YB_REQUIRE(p->n_anchors > 0 && p->n_anchors <= YB_MAX_ANCHORS && p->n_classes > 0, "decode_nms_tta: anchors/classes");
  YB_REQUIRE(p->max_det > 0 && p->max_det <= 4096, "decode_nms_tta: max_det must be in [1, 4096]");
  YB_REQUIRE(p->semantics >= 0 && p->semantics <= 2, "decode_nms_tta: bad semantics");
  int nl = 0;
  dtype = -1;
  dp.lvl_start[0] = 0;
  dp.pix_start[0] = 0;
  for (int q = 0; q < n_passes; ++q) {
    const yb_tta_pass& P = passes[q];
    YB_REQUIRE(P.n_levels >= 0 && P.n_levels <= YB_MAX_LEVELS, "decode_nms_tta: pass %d has %d levels", q, P.n_levels);
    YB_REQUIRE(P.scale > 0.f, "decode_nms_tta: pass %d scale must be positive", q);
    for (int l = 0; l < P.n_levels; ++l) {
      const yb_head_level& L = P.levels[l];
      if (dtype < 0) dtype = L.dtype;
      YB_REQUIRE(L.dtype == dtype && (dtype == YB_F16 || dtype == YB_BF16),
                 "decode_nms_tta: every level must hold fp16 (or every level bf16) logits");
      YB_REQUIRE(L.logits != nullptr && L.H > 0 && L.W > 0 && L.H <= 1023 && L.W <= 1023,
                 "decode_nms_tta: pass %d level %d empty or wider than 1023", q, l);
      // the row kernel's layout: NHWC rows of A*(nc+5) 16-bit logits, 16-byte aligned, at most 512 bytes
      YB_REQUIRE(L.stride_a == p->n_classes + 5 && L.stride_x % 8 == 0 && L.stride_x * 2 <= kRowMaxBytes &&
                     L.stride_x >= static_cast<long long>(p->n_anchors) * (p->n_classes + 5) && L.stride_y % 8 == 0 &&
                     L.stride_n % 8 == 0 && (reinterpret_cast<uintptr_t>(L.logits) & 15) == 0,
                 "decode_nms_tta: pass %d level %d is not an NHWC head buffer of <= 512-byte rows", q, l);
      dp.lvl[nl] = L;
      dp.scale[nl] = P.scale;
      dp.flip[nl] = P.flip_lr ? 1 : 0;
      dp.flip_w[nl] = P.canvas_w;
      dp.lvl_start[nl + 1] = dp.lvl_start[nl] + p->n_anchors * L.H * L.W;
      dp.pix_start[nl + 1] = dp.pix_start[nl] + L.H * L.W;
      ++nl;
    }
  }
  YB_REQUIRE(nl > 0, "decode_nms_tta: no levels");
  for (int l = nl; l < kTtaLevels; ++l) {
    dp.lvl[l] = dp.lvl[0];
    dp.scale[l] = 1.f;
    dp.flip[l] = 0;
    dp.flip_w[l] = 0.f;
    dp.lvl_start[l + 1] = dp.lvl_start[l];
    dp.pix_start[l + 1] = dp.pix_start[l];
  }
  apm = dp.lvl_start[nl];
  // the key's low word holds anchor * nc + class (unsigned); the NMS kernel indexes anchors with an int
  YB_REQUIRE(apm < (1ll << 31) && apm * p->n_classes < (1ll << 32),
             "decode_nms_tta: %lld anchors x %d classes overflow the 32-bit candidate index", apm, p->n_classes);
  dp.n_images = p->n_images;
  dp.n_levels = nl;
  dp.n_anchors = p->n_anchors;
  dp.n_classes = p->n_classes;
  dp.anchors_per_image = static_cast<int>(apm);
  dp.score_thresh = p->score_thresh;
  dp.cap_per_image = 0;
  return YB_OK;
}
}  // namespace

extern "C" size_t yb_decode_nms_tta_workspace_bytes(const yb_nms_params* p, int n_passes, const yb_tta_pass* passes) {
  TtaDecodeParams dp;
  int dtype;
  long long apm;
  if (fill_tta_params(p, n_passes, passes, dp, dtype, apm) != YB_OK) return 0;
  Workspace ws;
  const long long cap = (p->max_candidates + p->n_images - 1) / p->n_images;
  return carve(ws, nullptr, p->n_images, cap > 0 ? cap : 1, apm);
}

extern "C" int yb_decode_nms_tta(const yb_nms_params* p, int n_passes, const yb_tta_pass* passes,
                                 const float* rescale_dev, float* boxes_dev, float* scores_dev, int64_t* labels_dev,
                                 int32_t* counts_dev, int64_t* status_dev, void* workspace_dev, size_t workspace_bytes,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(boxes_dev && scores_dev && labels_dev && counts_dev && status_dev && workspace_dev,
             "decode_nms_tta: null output");
  TtaDecodeParams dp;
  int dtype;
  long long apm;
  int rc = fill_tta_params(p, n_passes, passes, dp, dtype, apm);
  if (rc != YB_OK) return rc;
  const long long cap = (p->max_candidates + p->n_images - 1) / p->n_images;
  YB_REQUIRE(cap >= 1, "decode_nms_tta: max_candidates too small");
  Workspace ws;
  const size_t need = carve(ws, static_cast<uint8_t*>(workspace_dev), p->n_images, cap, apm);
  if (need > workspace_bytes) {
    set_error("decode_nms_tta: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  dp.cap_per_image = cap;
  init_counters_kernel<<<(p->n_images + 127) / 128 + 1, 128, 0, stream>>>(ws, p->n_images,
                                                                          reinterpret_cast<long long*>(status_dev), 0);
  YB_CHECK_CUDA(cudaGetLastError());
  const int bpi = (dp.pix_start[dp.n_levels] + kRowWarps * kRowPixels - 1) / (kRowWarps * kRowPixels);
  const unsigned rblocks = static_cast<unsigned>(p->n_images) * static_cast<unsigned>(bpi);
  constexpr int kRowSmem = kRowWarps * kRowPixels * kRowPitch + kRowList * 8 + kRowWarps * kRowPairs * 8;
  static bool configured = false;
  if (!configured) {
    YB_CHECK_CUDA(cudaFuncSetAttribute(decode_rows_kernel<__half, TtaDecodeParams>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, kRowSmem));
    YB_CHECK_CUDA(cudaFuncSetAttribute(decode_rows_kernel<__nv_bfloat16, TtaDecodeParams>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, kRowSmem));
    configured = true;
  }
  if (dtype == YB_F16)
    decode_rows_kernel<__half, TtaDecodeParams><<<rblocks, kRowWarps * 32, kRowSmem, stream>>>(dp, ws, bpi);
  else
    decode_rows_kernel<__nv_bfloat16, TtaDecodeParams><<<rblocks, kRowWarps * 32, kRowSmem, stream>>>(dp, ws, bpi);
  YB_CHECK_CUDA(cudaGetLastError());
  return launch_nms(p, apm, cap, ws, rescale_dev, boxes_dev, scores_dev, labels_dev, counts_dev, status_dev, stream);
}
