// COCO box evaluation: pycocotools' evaluateImg + accumulate for iouType "bbox", reproduced bit for bit.
// "Rule n" refers to the numbered rules in oracle/restate_cocoeval.py.
//
//   append       update(): one thread per (row, slot) of a padded batch -> one 32-byte record
//   key1 / sort  records in (image, position) order (CUB radix sort, stable)
//   key2 / sort  stably by (category, -score): the accumulation order for every area and maxDets (rule 7)
//   gather       records in that order; per-category ranges
//   sort3        stably by image: each (image, category) is contiguous and in score order (rule 3)
//   heads        the first position of each (image, category) segment
//   npig         non-ignored GT per (category, area) with integer atomics (rule 7)
//   match        one CTA per segment, one warp per IoU threshold, greedy matching for the 4 areas (rules 5, 6)
//   accumulate   one CTA per (category, area, maxDets, threshold) (rule 7)
#include <cub/cub.cuh>

#include "common.cuh"

namespace yb {
namespace {

constexpr int kT = 10;        // IoU thresholds
constexpr int kR = 101;       // recall thresholds
constexpr int kA = 4;         // area ranges
constexpr int kM = 3;         // maxDets 1, 10, 100
constexpr int kMaxDet = 100;  // maxDets[-1]
constexpr int kMatchThreads = 32 * kT;
constexpr int kMatchGrid = 1024;
constexpr int kAccThreads = 256;
constexpr int kThreads = 256;

// params_dev: iouThrs[10] | recThrs[101] | areaRng[4][2]  (rule 1: computed by numpy on the host)
constexpr int kParRec = kT, kParArea = kT + kR;
static_assert(kT + kR + 2 * kA == YB_COCO_NUM_PARAMS, "params layout");

struct Ws {
  uint64_t *k_a, *k_b;
  int32_t *v_a, *v_b;
  int32_t *img, *cat, *rank;
  uint8_t* head;  // [n]: position i of the sort-3 order starts an (image, category) segment
  float* score;
  float4* box;
  uint8_t* bits;  // [n][kT]: bit a = matched to a GT with nonzero id, bit 4+a = dtIg, for area a
  int32_t *cat_start, *cat_end, *npig, *n_valid;
  uint32_t* gtm;  // matched-GT bitmaps, kMatchGrid x kT x kA x words
  void* cub;
  size_t cub_bytes;
};

inline size_t align_up(size_t x) { return (x + 255) & ~size_t(255); }

inline int bit_width(uint32_t x) {
  int b = 0;
  while (x) {
    ++b;
    x >>= 1;
  }
  return b;
}

inline int gtm_words(const yb_coco_gt* gt) { return (gt->max_gt_per_pair + 31) / 32 > 0 ? (gt->max_gt_per_pair + 31) / 32 : 1; }

size_t cub_bytes_needed(int n) {
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, n);
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, n);
  return std::max(a, b);
}

size_t carve(Ws& w, uint8_t* base, int n, const yb_coco_gt* gt) {
  size_t off = 0;
  auto take = [&](size_t bytes) -> uint8_t* {
    uint8_t* p = base ? base + off : nullptr;
    off += align_up(bytes);
    return p;
  };
  const size_t nn = n > 0 ? size_t(n) : 1;
  const size_t K = size_t(gt->n_categories);
  w.k_a = reinterpret_cast<uint64_t*>(take(nn * 8));
  w.k_b = reinterpret_cast<uint64_t*>(take(nn * 8));
  w.v_a = reinterpret_cast<int32_t*>(take(nn * 4));
  w.v_b = reinterpret_cast<int32_t*>(take(nn * 4));
  w.img = reinterpret_cast<int32_t*>(take(nn * 4));
  w.cat = reinterpret_cast<int32_t*>(take(nn * 4));
  w.rank = reinterpret_cast<int32_t*>(take(nn * 4));
  w.head = take(nn);
  w.score = reinterpret_cast<float*>(take(nn * 4));
  w.box = reinterpret_cast<float4*>(take(nn * 16));
  w.bits = take(nn * kT);
  // cat_start, cat_end, npig and n_valid are contiguous: one memset clears them
  w.cat_start = reinterpret_cast<int32_t*>(take((K * (2 + kA) + 1) * 4));
  w.cat_end = w.cat_start ? w.cat_start + K : nullptr;
  w.npig = w.cat_start ? w.cat_start + 2 * K : nullptr;
  w.n_valid = w.cat_start ? w.cat_start + (2 + kA) * K : nullptr;
  w.gtm = reinterpret_cast<uint32_t*>(take(size_t(kMatchGrid) * kT * kA * gtm_words(gt) * 4));
  w.cub_bytes = cub_bytes_needed(int(nn));
  w.cub = take(w.cub_bytes);
  return off;
}

__device__ __forceinline__ int warp_count(bool p) { return __popc(__ballot_sync(0xffffffffu, p)); }

// ---- append (rule 3: xyxy -> xywh in fp32) ----------------------------------------------------------
__global__ void __launch_bounds__(kThreads) coco_append_kernel(int n, int d, const float4* __restrict__ boxes,
                                                               const float* __restrict__ scores,
                                                               const int64_t* __restrict__ labels,
                                                               const int32_t* __restrict__ counts,
                                                               const int32_t* __restrict__ row_image,
                                                               const int32_t* __restrict__ label_map, int n_labels,
                                                               int4* __restrict__ out, int32_t* status) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= int64_t(n) * d) return;
  const int row = int(i / d), slot = int(i % d);
  const int img = row_image[row];
  int cat = -1;
  float score = 0.f;
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  if (img != YB_COCO_ROW_DROPPED && slot < counts[row]) {
    const int64_t l = labels[i];
    if (l < 0 || l >= n_labels) {
      atomicOr(status, YB_COCO_ST_BAD_LABEL);
    } else {
      cat = label_map[l];
    }
    if (img < 0) {
      atomicOr(status, YB_COCO_ST_UNKNOWN_IMAGE);
      cat = -1;
    }
    const float4 x = boxes[i];
    b = make_float4(x.x, x.y, __fsub_rn(x.z, x.x), __fsub_rn(x.w, x.y));
    score = scores[i];
  }
  out[2 * i] = make_int4(img, slot, cat, __float_as_int(score));
  out[2 * i + 1] = make_int4(__float_as_int(b.x), __float_as_int(b.y), __float_as_int(b.z), __float_as_int(b.w));
}

// ---- ordering ------------------------------------------------------------------------------------------
// Records with cat < 0 are not evaluated: their keys are all ones, so every sort leaves them at the end.
__global__ void __launch_bounds__(kThreads) coco_key1_kernel(const int4* __restrict__ rec, int n, Ws w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < n;
  const int4 m = in ? rec[2 * i] : make_int4(0, 0, -1, 0);
  const bool valid = in && m.z >= 0;
  if (in) {
    w.k_a[i] = valid ? (uint64_t(uint32_t(m.x)) << 32 | uint32_t(m.y)) : ~0ull;
    w.v_a[i] = i;
  }
  const int c = warp_count(valid);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(w.n_valid, c);
}

__device__ __forceinline__ uint32_t descending_score_key(float s) {
  if (s == 0.f) s = 0.f;  // -0 and +0 tie, as in numpy's comparison sort
  const uint32_t u = __float_as_uint(s);
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}

__global__ void __launch_bounds__(kThreads) coco_key2_kernel(const int4* __restrict__ rec, int n, Ws w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = w.v_b[i];
  const int4 m = rec[2 * r];
  w.k_a[i] = m.z >= 0 ? (uint64_t(uint32_t(m.z)) << 32 | descending_score_key(__int_as_float(m.w))) : ~0ull;
  w.v_a[i] = r;
}

// After sort 2, v_b holds the records in accumulation order; position j of that order is a detection's index
// in every later array.
__global__ void __launch_bounds__(kThreads) coco_gather_kernel(const int4* __restrict__ rec, int n, Ws w) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int nv = *w.n_valid;
  uint32_t* key3 = reinterpret_cast<uint32_t*>(w.k_a);
  w.v_a[j] = j;
  if (j >= nv) {
    key3[j] = ~0u;
    return;
  }
  const int r = w.v_b[j];
  const int4 m = rec[2 * r];
  const int4 b = rec[2 * r + 1];
  w.img[j] = m.x;
  w.cat[j] = m.z;
  w.score[j] = __int_as_float(m.w);
  w.box[j] = make_float4(__int_as_float(b.x), __int_as_float(b.y), __int_as_float(b.z), __int_as_float(b.w));
  key3[j] = uint32_t(m.x);
  if (j == 0 || rec[2 * w.v_b[j - 1]].z != m.z) w.cat_start[m.z] = j;
  if (j == nv - 1 || rec[2 * w.v_b[j + 1]].z != m.z) w.cat_end[m.z] = j + 1;
}

// After sort 3, v_b lists positions grouped by (image, category), each group in accumulation order.
__global__ void __launch_bounds__(kThreads) coco_heads_kernel(int n, Ws w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int head = 0;
  if (i < *w.n_valid) {
    const int j = w.v_b[i];
    head = i == 0 || w.img[j] != w.img[w.v_b[i - 1]] || w.cat[j] != w.cat[w.v_b[i - 1]];
  }
  w.head[i] = uint8_t(head);
}

// ---- GT: npig per (category, area) over the evaluated images (rules 4, 7) -----------------------------
__global__ void __launch_bounds__(kThreads) coco_npig_kernel(yb_coco_gt gt, const uint8_t* __restrict__ evaluated,
                                                             const double* __restrict__ par, Ws w) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= gt.n_gt || !evaluated[gt.gt_img[g]] || (gt.gt_flags[g] & YB_COCO_GT_CROWD)) return;
  const double area = gt.gt_area[g];
  for (int a = 0; a < kA; ++a)
    if (!(area < par[kParArea + 2 * a] || area > par[kParArea + 2 * a + 1])) atomicAdd(&w.npig[gt.gt_cat[g] * kA + a], 1);
}

// ---- matching (rules 5, 6) -------------------------------------------------------------------------
// pycocotools' bbIou in float64, every operation rounded on its own (no FMA contraction).
__device__ __forceinline__ double box_iou(double dx, double dy, double dw, double dh, double da, double gx, double gy,
                                          double gw, double gh, bool crowd) {
  const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(gw, gx)), fmax(dx, gx));
  if (w <= 0.0) return 0.0;
  const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(gh, gy)), fmax(dy, gy));
  if (h <= 0.0) return 0.0;
  const double i = __dmul_rn(w, h);
  const double u = crowd ? da : __dsub_rn(__dadd_rn(da, __dmul_rn(gw, gh)), i);
  return __ddiv_rn(i, u);
}

__device__ __forceinline__ int lower_bound_cat(const int32_t* cat, int lo, int hi, int k) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cat[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// One CTA per (image, category) segment (a grid-stride walk over the segments' first positions); warp t runs the greedy sequences of IoU threshold t for the
// four area ranges over the first 100 detections.  GT stay in file order: the non-ignored ones of an area form the
// first search segment and the ignored ones the second, which is pycocotools' stable sort by gtIg plus its `break`.
__global__ void __launch_bounds__(kMatchThreads) coco_match_kernel(yb_coco_gt gt, const double* __restrict__ par,
                                                                    int words, Ws w) {
  const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const double thr = fmin(par[t], 1.0 - 1e-10);
  double lo[kA], hi[kA];
#pragma unroll
  for (int a = 0; a < kA; ++a) {
    lo[a] = par[kParArea + 2 * a];
    hi[a] = par[kParArea + 2 * a + 1];
  }
  uint32_t* gtm = w.gtm + (size_t(blockIdx.x) * kT + t) * kA * words;
  const int nv = *w.n_valid;
  for (int i0 = blockIdx.x; i0 < nv; i0 += gridDim.x) {
    if (!w.head[i0]) continue;
    int i1 = i0 + 1;
    while (i1 < nv && !w.head[i1]) ++i1;
    const int j0 = w.v_b[i0];
    const int img = w.img[j0], cat = w.cat[j0];
    if (t == 0)
      for (int i = i0 + lane; i < i1; i += 32) w.rank[w.v_b[i]] = i - i0;
    const int g0 = lower_bound_cat(gt.gt_cat, gt.img_start[img], gt.img_start[img + 1], cat);
    const int G = lower_bound_cat(gt.gt_cat, g0, gt.img_start[img + 1], cat + 1) - g0;
    for (int x = lane; x < kA * words; x += 32) gtm[x] = 0u;
    __syncwarp();
    const int nd = min(i1 - i0, kMaxDet);
    for (int d = 0; d < nd; ++d) {
      const int j = w.v_b[i0 + d];
      const float4 b = w.box[j];
      const double dx = b.x, dy = b.y, dw = b.z, dh = b.w;
      const double da = __dmul_rn(dw, dh);
      double best[kA][2];
      int bg[kA][2];
#pragma unroll
      for (int a = 0; a < kA; ++a) best[a][0] = best[a][1] = -1.0, bg[a][0] = bg[a][1] = -1;
      for (int g = lane; g < G; g += 32) {
        const int gi = g0 + g;
        const bool crowd = gt.gt_flags[gi] & YB_COCO_GT_CROWD;
        const double2 gxy = reinterpret_cast<const double2*>(gt.gt_box)[2 * gi];
        const double2 gwh = reinterpret_cast<const double2*>(gt.gt_box)[2 * gi + 1];
        const double iou = box_iou(dx, dy, dw, dh, da, gxy.x, gxy.y, gwh.x, gwh.y, crowd);
        if (!(iou >= thr)) continue;
        const double area = gt.gt_area[gi];
#pragma unroll
        for (int a = 0; a < kA; ++a) {
          const bool taken = !crowd && ((gtm[a * words + (g >> 5)] >> lane) & 1u);
          const bool ig = crowd || area < lo[a] || area > hi[a];
          // lanes visit g in ascending order: >= keeps the last index of the maximum (rule 6)
          if (!taken && !ig && iou >= best[a][0]) best[a][0] = iou, bg[a][0] = g;
          if (!taken && ig && iou >= best[a][1]) best[a][1] = iou, bg[a][1] = g;
        }
      }
      uint32_t byte = 0;
#pragma unroll
      for (int a = 0; a < kA; ++a) {
#pragma unroll
        for (int s2 = 0; s2 < 2; ++s2) {
#pragma unroll
          for (int off = 16; off; off >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best[a][s2], off);
            const int og = __shfl_xor_sync(0xffffffffu, bg[a][s2], off);
            if (ob > best[a][s2] || (ob == best[a][s2] && og > bg[a][s2])) best[a][s2] = ob, bg[a][s2] = og;
          }
        }
        const bool ig = bg[a][0] < 0;  // the ignored GT only when no non-ignored one qualified
        const int m = ig ? bg[a][1] : bg[a][0];
        const bool id_nonzero = m >= 0 && (gt.gt_flags[g0 + m] & YB_COCO_GT_ID_NONZERO);
        bool dt_ig = m >= 0 && ig;
        if (!id_nonzero && (da < lo[a] || da > hi[a])) dt_ig = true;
        byte |= uint32_t(id_nonzero) << a | uint32_t(dt_ig) << (4 + a);
        if (m >= 0 && lane == (m & 31)) gtm[a * words + (m >> 5)] |= 1u << lane;
      }
      __syncwarp();
      if (lane == 0) w.bits[size_t(j) * kT + t] = uint8_t(byte);
    }
    __syncwarp();
  }
}

// ---- accumulation (rule 7) -----------------------------------------------------------------------------
struct Counts3 {
  int n, tp, fp;
};
__device__ __forceinline__ Counts3 operator+(const Counts3& x, const Counts3& y) {
  return Counts3{x.n + y.n, x.tp + y.tp, x.fp + y.fp};
}

// One CTA per (category k, area a, maxDets m, threshold t), streaming category k's detections in accumulation order.
// For recall threshold r, searchsorted(rc, r) is the first position whose cumulative tp reaches T_r, the least
// integer c with c / npig >= r.  A position with cumulative tp c belongs to bucket b = max{r : T_r <= c}, so the
// suffix maximum of pr from that position is the maximum over the buckets >= r: one pass, no per-CTA arrays.
__global__ void __launch_bounds__(kAccThreads) coco_accumulate_kernel(int K, const double* __restrict__ par, Ws w,
                                                                       double* __restrict__ precision,
                                                                       double* __restrict__ recall,
                                                                       double* __restrict__ scores) {
  using Scan = cub::BlockScan<Counts3, kAccThreads>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int T[kR];
  __shared__ unsigned long long bucket[kR];
  __shared__ double sc[kR];
  __shared__ Counts3 carry;
  const int t = blockIdx.x % kT;
  const int mi = (blockIdx.x / kT) % kM;
  const int a = (blockIdx.x / (kT * kM)) % kA;
  const int k = blockIdx.x / (kT * kM * kA);
  const int maxdet = mi == 0 ? 1 : (mi == 1 ? 10 : kMaxDet);
  const int npig = w.npig[k * kA + a];
  auto p_at = [&](int r) { return ((((size_t(t) * kR + r) * K + k) * kA + a) * kM + mi); };
  const size_t rec_at = ((size_t(t) * K + k) * kA + a) * kM + mi;
  if (npig == 0) {
    for (int r = threadIdx.x; r < kR; r += blockDim.x) precision[p_at(r)] = -1.0, scores[p_at(r)] = -1.0;
    if (threadIdx.x == 0) recall[rec_at] = -1.0;
    return;
  }
  const double np_d = double(npig);
  if (threadIdx.x < kR) {
    const double r = par[kParRec + threadIdx.x];
    int c = max(0, int(floor(r * np_d)) - 1);  // c / npig < r here; step up to the first c that reaches r
    while (c < npig && !(__ddiv_rn(double(c), np_d) >= r)) ++c;
    T[threadIdx.x] = c;
    bucket[threadIdx.x] = 0ull;  // +0.0: pr is never negative
    sc[threadIdx.x] = 0.0;
  }
  if (threadIdx.x == 0) carry = Counts3{0, 0, 0};
  __syncthreads();
  const int cs = w.cat_start[k], ce = w.cat_end[k];
  for (int base = cs; base < ce; base += kAccThreads) {
    const int i = base + threadIdx.x;
    const bool inc = i < ce && w.rank[i] < maxdet;
    uint32_t byte = inc ? w.bits[size_t(i) * kT + t] : 0u;
    const bool matched = (byte >> a) & 1u, ig = (byte >> (4 + a)) & 1u;
    const Counts3 in{int(inc), int(inc && matched && !ig), int(inc && !matched && !ig)};
    Counts3 pre, agg;
    Scan(scan_tmp).InclusiveSum(in, pre, agg);
    const Counts3 c0 = carry;
    if (inc) {
      const int tp = c0.tp + pre.tp, fp = c0.fp + pre.fp, pos = c0.n + pre.n;  // pos is 1-based
      const double tpd = double(tp);
      const double pr = __ddiv_rn(tpd, __dadd_rn(__dadd_rn(double(fp), tpd), 2.220446049250313e-16));
      int lo = 0, hi = kR;  // bucket: last r with T[r] <= tp
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (T[mid] <= tp) lo = mid + 1;
        else hi = mid;
      }
      if (lo > 0) atomicMax(&bucket[lo - 1], static_cast<unsigned long long>(__double_as_longlong(pr)));
      // the position searchsorted gives for r: the first one (T_r == 0) or the one where tp reaches T_r
      const int key = in.tp ? tp : (pos == 1 ? 0 : -1);
      if (key >= 0) {
        const double s = double(w.score[i]);
        for (int r = 0; r < kR && T[r] <= key; ++r)
          if (T[r] == key || (pos == 1 && T[r] == 0)) sc[r] = s;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) carry = c0 + agg;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const Counts3 tot = carry;
    double run = 0.0;
    for (int r = kR - 1; r >= 0; --r) {
      run = fmax(run, __longlong_as_double(static_cast<long long>(bucket[r])));
      const bool reached = tot.n > 0 && T[r] <= tot.tp;
      precision[p_at(r)] = reached ? run : 0.0;
      scores[p_at(r)] = reached ? sc[r] : 0.0;
    }
    recall[rec_at] = tot.n > 0 ? __ddiv_rn(double(tot.tp), np_d) : 0.0;
  }
}

inline unsigned blocks(int64_t n) { return unsigned((n + kThreads - 1) / kThreads); }

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_coco_append(int n, int d, const float* boxes_dev, const float* scores_dev, const int64_t* labels_dev,
                              const int32_t* counts_dev, const int32_t* row_image_dev, const int32_t* label_map_dev,
                              int32_t n_labels, int32_t* records_dev, int32_t* status_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(n >= 0 && d >= 0 && int64_t(n) * d < (1ll << 31), "coco_append: n x d out of range");
  if (int64_t(n) * d == 0) return YB_OK;
  YB_REQUIRE(boxes_dev && scores_dev && labels_dev && counts_dev && row_image_dev && records_dev && status_dev,
             "coco_append: null argument");
  YB_REQUIRE(n_labels >= 0 && (n_labels == 0 || label_map_dev), "coco_append: bad label map");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(boxes_dev) & 15) == 0 && (reinterpret_cast<uintptr_t>(records_dev) & 15) == 0,
             "coco_append: boxes and records must be 16-byte aligned");
  coco_append_kernel<<<blocks(int64_t(n) * d), kThreads, 0, stream>>>(
      n, d, reinterpret_cast<const float4*>(boxes_dev), scores_dev, labels_dev, counts_dev, row_image_dev,
      label_map_dev, n_labels, reinterpret_cast<int4*>(records_dev), status_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" size_t yb_coco_evaluate_workspace_bytes(int64_t n_records, const yb_coco_gt* gt) {
  if (!gt || n_records < 0 || n_records >= (1ll << 31)) return 0;
  Ws w;
  return carve(w, nullptr, int(n_records), gt);
}

extern "C" int yb_coco_evaluate(const yb_coco_gt* gt, const int32_t* records_dev, int64_t n_records,
                                const uint8_t* evaluated_dev, const double* params_dev, double* precision_dev,
                                double* recall_dev, double* scores_dev, void* workspace_dev, size_t workspace_bytes,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  YB_REQUIRE(gt && params_dev && precision_dev && recall_dev && scores_dev && workspace_dev && evaluated_dev,
             "coco_evaluate: null argument");
  YB_REQUIRE(n_records >= 0 && n_records < (1ll << 31), "coco_evaluate: n_records out of range");
  YB_REQUIRE(n_records == 0 || records_dev, "coco_evaluate: null records");
  YB_REQUIRE(gt->n_images >= 0 && gt->n_categories > 0 && gt->n_gt >= 0 && gt->max_gt_per_pair >= 0,
             "coco_evaluate: bad GT descriptor");
  YB_REQUIRE(gt->img_start && (gt->n_gt == 0 || (gt->gt_img && gt->gt_cat && gt->gt_box && gt->gt_area && gt->gt_flags)),
             "coco_evaluate: null GT array");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(records_dev) & 15) == 0 && (reinterpret_cast<uintptr_t>(gt->gt_box) & 15) == 0,
             "coco_evaluate: records and GT boxes must be 16-byte aligned");
  const int n = int(n_records);
  const int K = gt->n_categories;
  Ws w;
  const size_t need = carve(w, static_cast<uint8_t*>(workspace_dev), n, gt);
  if (need > workspace_bytes) {
    set_error("coco_evaluate: workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    return YB_ERR_WORKSPACE;
  }
  const int4* rec = reinterpret_cast<const int4*>(records_dev);
  YB_CHECK_CUDA(cudaMemsetAsync(w.cat_start, 0, (size_t(K) * (2 + kA) + 1) * 4, stream));
  if (gt->n_gt > 0) {
    coco_npig_kernel<<<blocks(gt->n_gt), kThreads, 0, stream>>>(*gt, evaluated_dev, params_dev, w);
    YB_CHECK_CUDA(cudaGetLastError());
  }
  if (n > 0) {
    const int img_bits = 32 + bit_width(uint32_t(gt->n_images));
    const int cat_bits = 32 + bit_width(uint32_t(K));
    coco_key1_kernel<<<blocks(n), kThreads, 0, stream>>>(rec, n, w);
    YB_CHECK_CUDA(cudaGetLastError());
    size_t tb = w.cub_bytes;
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, tb, w.k_a, w.k_b, w.v_a, w.v_b, n, 0, img_bits, stream));
    coco_key2_kernel<<<blocks(n), kThreads, 0, stream>>>(rec, n, w);
    YB_CHECK_CUDA(cudaGetLastError());
    tb = w.cub_bytes;
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, tb, w.k_a, w.k_b, w.v_a, w.v_b, n, 0, cat_bits, stream));
    coco_gather_kernel<<<blocks(n), kThreads, 0, stream>>>(rec, n, w);
    YB_CHECK_CUDA(cudaGetLastError());
    tb = w.cub_bytes;
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, tb, reinterpret_cast<const uint32_t*>(w.k_a),
                                                  reinterpret_cast<uint32_t*>(w.k_b), w.v_a, w.v_b, n, 0,
                                                  std::max(1, bit_width(uint32_t(gt->n_images))), stream));
    coco_heads_kernel<<<blocks(n), kThreads, 0, stream>>>(n, w);
    YB_CHECK_CUDA(cudaGetLastError());
    coco_match_kernel<<<unsigned(std::min(n, kMatchGrid)), kMatchThreads, 0, stream>>>(*gt, params_dev,
                                                                                       gtm_words(gt), w);
    YB_CHECK_CUDA(cudaGetLastError());
  }
  coco_accumulate_kernel<<<unsigned(K * kA * kM * kT), kAccThreads, 0, stream>>>(K, params_dev, w, precision_dev,
                                                                                  recall_dev, scores_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
