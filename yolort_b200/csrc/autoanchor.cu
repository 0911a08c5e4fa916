// YOLOv5's AutoAnchor (yolort/v5/utils/autoanchor.py) on the device: the anchor metric, scipy's k-means and the
// genetic anchor evolution.  Every random draw was made on the host (yolort_b200/v5/utils/autoanchor.py); these
// kernels do the arithmetic, restated step by step in oracle/restate_autoanchor.py.
//
//   aa_metric_kernel       ratio metric of every label against the anchors (float32 or float64, as torch promotes):
//                          per-block counts and float64 sums, folded by aa_metric_fold_kernel in block order
//   km_vq_kernel           scipy's vq for every live trial: squared distances in IEEE double, first minimum, sqrt
//   km_mean_kernel         numpy's pairwise mean of the distances (the tree of pairwise_sum, seeded with 0.0) and
//                          _kmeans' stopping rule; one block per trial
//   km_update_kernel       update_cluster_means: per (trial, cluster), members in observation order, one dependent
//                          double chain per dimension, then / count
//   km_compact_kernel      code_book[has_members]
//   aa_evolve_kernel       all generations in one cooperative launch: per generation the mutated anchors, the
//                          per-label float32 fitness terms, an exact fixed-point sum and one grid barrier
//
// Built with -fmad=false (Makefile) and written with _rn intrinsics: no product is contracted into an FMA.
#include <cooperative_groups.h>

#include <cmath>
#include <vector>

#include "common.cuh"
#include <math_constants.h>

namespace cg = cooperative_groups;

namespace yb {
namespace {

constexpr int kThreads = 256;
constexpr int kMeanThreads = 512;

// ---- metric -----------------------------------------------------------------------------------------------------
// part[b] = {count best > thr, count x > thr, sum x, sum best, sum x[x > thr]} of block b's labels
struct MetricPart {
  long long n_best, n_x;
  double s_x, s_best, s_past;
};

template <bool F64>
__global__ void __launch_bounds__(kThreads) aa_metric_kernel(const float2* __restrict__ wh, int64_t n, const double* anchors,
                                                             int na, double thr, MetricPart* part) {
  __shared__ double sa[2 * YB_AA_MAX_ANCHORS];
  __shared__ MetricPart sp[kThreads / 32];
  for (int j = threadIdx.x; j < 2 * na; j += blockDim.x) sa[j] = anchors[j];
  __syncthreads();
  const float thr32 = float(thr);
  MetricPart p{0, 0, 0.0, 0.0, 0.0};
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const float2 w = wh[i];
    double best = 0.0;
    for (int j = 0; j < na; ++j) {
      double x;
      bool past;
      if (F64) {
        const double r0 = __ddiv_rn(double(w.x), sa[2 * j]), r1 = __ddiv_rn(double(w.y), sa[2 * j + 1]);
        x = fmin(fmin(r0, __ddiv_rn(1.0, r0)), fmin(r1, __ddiv_rn(1.0, r1)));
        past = x > thr;
      } else {
        const float r0 = __fdiv_rn(w.x, float(sa[2 * j])), r1 = __fdiv_rn(w.y, float(sa[2 * j + 1]));
        const float xf = fminf(fminf(r0, __fdiv_rn(1.0f, r0)), fminf(r1, __fdiv_rn(1.0f, r1)));
        x = xf;
        past = xf > thr32;
      }
      best = j == 0 ? x : fmax(best, x);
      p.s_x += x;
      if (past) {
        p.n_x += 1;
        p.s_past += x;
      }
    }
    p.s_best += best;
    p.n_best += F64 ? (best > thr) : (float(best) > thr32);
  }
  // fixed-shape tree: warp shuffles, then warp 0 over the warps, so a replay adds in the same order
  for (int o = 16; o > 0; o >>= 1) {
    p.n_best += __shfl_down_sync(0xffffffffu, p.n_best, o);
    p.n_x += __shfl_down_sync(0xffffffffu, p.n_x, o);
    p.s_x += __shfl_down_sync(0xffffffffu, p.s_x, o);
    p.s_best += __shfl_down_sync(0xffffffffu, p.s_best, o);
    p.s_past += __shfl_down_sync(0xffffffffu, p.s_past, o);
  }
  if ((threadIdx.x & 31) == 0) sp[threadIdx.x >> 5] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    MetricPart t = sp[0];
    for (int w = 1; w < kThreads / 32; ++w) {
      t.n_best += sp[w].n_best;
      t.n_x += sp[w].n_x;
      t.s_x += sp[w].s_x;
      t.s_best += sp[w].s_best;
      t.s_past += sp[w].s_past;
    }
    part[blockIdx.x] = t;
  }
}

__global__ void aa_metric_fold_kernel(const MetricPart* part, int n_parts, long long* counts, double* sums) {
  if (threadIdx.x != 0) return;
  MetricPart t{0, 0, 0.0, 0.0, 0.0};
  for (int b = 0; b < n_parts; ++b) {
    t.n_best += part[b].n_best;
    t.n_x += part[b].n_x;
    t.s_x += part[b].s_x;
    t.s_best += part[b].s_best;
    t.s_past += part[b].s_past;
  }
  counts[0] = t.n_best;
  counts[1] = t.n_x;
  sums[0] = t.s_x;
  sums[1] = t.s_best;
  sums[2] = t.s_past;
}

// ---- k-means ----------------------------------------------------------------------------------------------------
enum : int { kRun = 0, kFinal = 1, kDone = 2 };

struct TrialState {
  int phase;       // kRun: the next vq + mean is an iteration; kFinal: it gives the final distortion; kDone
  int ncb;         // codes in the book
  int update;      // the update kernel runs after this mean
  int pad;
  double prev;     // the previous iteration's mean distortion (inf before the first)
};

// One node of numpy's pairwise_sum tree over n elements: a leaf sums [lo, lo + len) with 8 accumulators (or one, below
// 8 elements); an inner node adds its two children.
struct SumNode {
  int64_t lo;
  int32_t len, left, right, pad;
};

__global__ void __launch_bounds__(kThreads) km_vq_kernel(const double2* __restrict__ obs, int64_t n, const double* books,
                                                        int k, const TrialState* st, uint8_t* codes, double* dist) {
  const int t = blockIdx.y;
  const TrialState s = st[t];
  if (s.phase == kDone) return;
  __shared__ double2 cb[YB_AA_MAX_ANCHORS];
  for (int j = threadIdx.x; j < s.ncb; j += blockDim.x) cb[j] = make_double2(books[(t * k + j) * 2], books[(t * k + j) * 2 + 1]);
  __syncthreads();
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const double2 o = obs[i];
    double low = CUDART_INF;
    int code = 0;
    for (int j = 0; j < s.ncb; ++j) {
      const double d0 = __dsub_rn(cb[j].x, o.x), d1 = __dsub_rn(cb[j].y, o.y);
      const double d = __dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1));
      if (d < low) {
        low = d;
        code = j;
      }
    }
    codes[t * n + i] = uint8_t(code);
    dist[t * n + i] = __dsqrt_rn(low);
  }
}

__global__ void __launch_bounds__(kMeanThreads) km_mean_kernel(const double* dist, int64_t n, const SumNode* nodes,
                                                              const int* depth_start, int depths,
                                                              double* node_val, double thresh, TrialState* st,
                                                              double* dist_out, int* live) {
  const int t = blockIdx.x;
  if (st[t].phase == kDone) return;
  const double* a = dist + t * n;
  double* val = node_val + int64_t(t) * depth_start[depths];
  // every leaf first, then the inner nodes depth by depth from the deepest up
  for (int l = threadIdx.x; l < depth_start[depths]; l += blockDim.x) {
    const SumNode nd = nodes[l];
    if (nd.left >= 0) continue;
    const double* p = a + nd.lo;
    double res;
    if (nd.len < 8) {
      res = 0.0;
      for (int i = 0; i < nd.len; ++i) res = __dadd_rn(res, p[i]);
    } else {
      double r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = p[j];
      int i = 8;
      for (; i < nd.len - (nd.len % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], p[i + j]);
      }
      res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                      __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
      for (; i < nd.len; ++i) res = __dadd_rn(res, p[i]);
    }
    val[l] = res;
  }
  __syncthreads();
  for (int d = depths - 1; d >= 0; --d) {
    for (int q = depth_start[d] + threadIdx.x; q < depth_start[d + 1]; q += blockDim.x) {
      const SumNode nd = nodes[q];
      if (nd.left >= 0) val[q] = __dadd_rn(val[nd.left], val[nd.right]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double cur = __ddiv_rn(__dadd_rn(0.0, val[0]), double(n));
    TrialState s = st[t];
    if (s.phase == kFinal) {
      dist_out[t] = cur;
      s.phase = kDone;
      s.update = 0;
      atomicSub(live, 1);
    } else {
      const double diff = fabs(s.prev - cur);
      s.prev = cur;
      s.update = 1;
      if (!(diff > thresh)) s.phase = kFinal;
    }
    st[t] = s;
  }
}

__global__ void __launch_bounds__(kThreads) km_update_kernel(const double2* __restrict__ obs, int64_t n,
                                                            const uint8_t* codes, int k, const TrialState* st,
                                                            double* sums, long long* counts) {
  const int c = blockIdx.x, t = blockIdx.y;
  const TrialState s = st[t];
  if (!s.update || c >= s.ncb) return;
  __shared__ double2 buf[kThreads];
  __shared__ int warp_n[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double sx = 0.0, sy = 0.0;
  long long cnt = 0;
  const uint8_t* cd = codes + t * n;
  for (int64_t base = 0; base < n; base += kThreads) {
    const int64_t i = base + threadIdx.x;
    const bool mine = i < n && cd[i] == c;
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) warp_n[warp] = __popc(m);
    __syncthreads();
    int off = 0, tot = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      off += w < warp ? warp_n[w] : 0;
      tot += warp_n[w];
    }
    if (mine) buf[off + __popc(m & ((1u << lane) - 1u))] = obs[i];
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int q = 0; q < tot; ++q) {     // observation order: scipy's update_cluster_means loop
        sx = __dadd_rn(sx, buf[q].x);
        sy = __dadd_rn(sy, buf[q].y);
      }
      cnt += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int q = t * k + c;
    counts[q] = cnt;
    if (cnt > 0) {
      sums[2 * q] = __ddiv_rn(sx, double(cnt));
      sums[2 * q + 1] = __ddiv_rn(sy, double(cnt));
    }
  }
}

__global__ void km_compact_kernel(const double* sums, const long long* counts, int k, TrialState* st, double* books) {
  const int t = blockIdx.x;
  if (threadIdx.x != 0 || !st[t].update) return;
  int m = 0;
  for (int c = 0; c < st[t].ncb; ++c) {
    if (counts[t * k + c] > 0) {
      books[(t * k + m) * 2] = sums[(t * k + c) * 2];
      books[(t * k + m) * 2 + 1] = sums[(t * k + c) * 2 + 1];
      ++m;
    }
  }
  st[t].ncb = m;
  st[t].update = 0;
}

// ---- evolution --------------------------------------------------------------------------------------------------
// sums[g + 1]: the fixed-point sum of generation g (sums[0]: the starting anchors); every block adds its part with one
// atomic, and after the grid barrier every block reads the same total and takes the same decision.
__global__ void __launch_bounds__(kThreads) aa_evolve_kernel(const float2* __restrict__ wh, int64_t n, int na,
                                                            const double* k0, const double* v, int gen, float thr,
                                                            double unit, unsigned long long* sums, float* fit,
                                                            uint8_t* accepted, double* k_out) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double k[2 * YB_AA_MAX_ANCHORS];
  __shared__ double kg[2 * YB_AA_MAX_ANCHORS];
  __shared__ float kg32[2 * YB_AA_MAX_ANCHORS];
  __shared__ unsigned long long warp_s[kThreads / 32];
  for (int j = threadIdx.x; j < 2 * na; j += blockDim.x) k[j] = k0[j];
  const float fn = float(n);           // torch's mean: the float32 sum / numel, in float32
  float f = 0.0f;
  for (int g = -1; g < gen; ++g) {
    __syncthreads();
    for (int j = threadIdx.x; j < 2 * na; j += blockDim.x) {
      double x = k[j];
      if (g >= 0) {
        x = __dmul_rn(x, v[int64_t(g) * 2 * na + j]);
        x = x < 2.0 ? 2.0 : x;        // clip(min=2.0)
      }
      kg[j] = x;
      kg32[j] = __double2float_rn(x);
    }
    __syncthreads();
    unsigned long long part = 0;
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
      const float2 w = wh[i];
      float best = 0.0f;
      for (int j = 0; j < na; ++j) {
        const float r0 = __fdiv_rn(w.x, kg32[2 * j]), r1 = __fdiv_rn(w.y, kg32[2 * j + 1]);
        const float x = fminf(fminf(r0, __fdiv_rn(1.0f, r0)), fminf(r1, __fdiv_rn(1.0f, r1)));
        best = j == 0 ? x : fmaxf(best, x);
      }
      // best in (thr, 1] is a whole multiple of unit: the product is an exact integer
      if (best > thr) part += (unsigned long long)__dmul_rn(double(best), 1.0 / unit);
    }
    for (int o = 16; o > 0; o >>= 1) part += __shfl_down_sync(0xffffffffu, part, o);
    if ((threadIdx.x & 31) == 0) warp_s[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long b = 0;
      for (int w = 0; w < kThreads / 32; ++w) b += warp_s[w];
      if (b) atomicAdd(sums + (g + 1), b);
    }
    grid.sync();
    const unsigned long long total = __ldcg(sums + (g + 1));
    const float fg = __fdiv_rn(__double2float_rn(__dmul_rn(double(total), unit)), fn);
    if (g < 0) {
      f = fg;
    } else if (fg > f) {
      f = fg;
      for (int j = threadIdx.x; j < 2 * na; j += blockDim.x) k[j] = kg[j];
      if (blockIdx.x == 0 && threadIdx.x == 0) accepted[g] = 1;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) fit[g + 1] = f;
  }
  __syncthreads();
  if (blockIdx.x == 0)
    for (int j = threadIdx.x; j < 2 * na; j += blockDim.x) k_out[j] = k[j];
}

// numpy's pairwise_sum tree over n elements, nodes ordered by depth; *depth_start gets depths + 1 offsets
void build_sum_tree(int64_t n, std::vector<SumNode>& nodes, std::vector<int>& depth_start) {
  struct Item {
    int64_t lo, len;
    int parent, side;
  };
  std::vector<Item> level{{0, n, -1, 0}};
  while (!level.empty()) {
    depth_start.push_back(int(nodes.size()));
    std::vector<Item> next;
    for (const Item& it : level) {
      const int id = int(nodes.size());
      nodes.push_back(SumNode{it.lo, int32_t(it.len), -1, -1, 0});
      if (it.parent >= 0) (it.side ? nodes[it.parent].right : nodes[it.parent].left) = id;
      if (it.len > 128) {
        int64_t n2 = it.len / 2;
        n2 -= n2 % 8;
        next.push_back({it.lo, n2, id, 0});
        next.push_back({it.lo + n2, it.len - n2, id, 1});
      }
    }
    level.swap(next);
  }
  depth_start.push_back(int(nodes.size()));
}

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

struct KmLayout {
  size_t codes, dist, node_val, nodes, depth, state, sums, counts, live, total;
  int n_nodes, depths;
};

KmLayout km_layout(int64_t n, int k, int trials) {
  std::vector<SumNode> nodes;
  std::vector<int> ds;
  build_sum_tree(n, nodes, ds);
  KmLayout L{};
  L.n_nodes = int(nodes.size());
  L.depths = int(ds.size()) - 1;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += align256(bytes);
    return o;
  };
  L.codes = take(size_t(trials) * n);
  L.dist = take(size_t(trials) * n * sizeof(double));
  L.node_val = take(size_t(trials) * L.n_nodes * sizeof(double));
  L.nodes = take(size_t(L.n_nodes) * sizeof(SumNode));
  L.depth = take(ds.size() * sizeof(int));
  L.state = take(size_t(trials) * sizeof(TrialState));
  L.sums = take(size_t(trials) * k * 2 * sizeof(double));
  L.counts = take(size_t(trials) * k * sizeof(long long));
  L.live = take(sizeof(int));
  L.total = off;
  return L;
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_anchor_metric(const float* wh_dev, int64_t n, const double* anchors_dev, int n_anchors, int f64,
                                double thr, int64_t* counts_dev, double* sums_dev, void* workspace,
                                size_t workspace_bytes, void* stream_) {
  YB_REQUIRE(wh_dev && anchors_dev && counts_dev && sums_dev && workspace, "anchor_metric: null argument");
  YB_REQUIRE(n > 0 && n_anchors >= 1 && n_anchors <= YB_AA_MAX_ANCHORS, "anchor_metric: %lld labels, %d anchors",
             (long long)n, n_anchors);
  YB_REQUIRE(workspace_bytes >= YB_AA_METRIC_WORKSPACE, "anchor_metric: workspace of %zu bytes", workspace_bytes);
  const int blocks = int(std::min<int64_t>((n + kThreads - 1) / kThreads, YB_AA_METRIC_WORKSPACE / sizeof(MetricPart)));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MetricPart* part = static_cast<MetricPart*>(workspace);
  const float2* wh = reinterpret_cast<const float2*>(wh_dev);
  if (f64)
    aa_metric_kernel<true><<<blocks, kThreads, 0, stream>>>(wh, n, anchors_dev, n_anchors, thr, part);
  else
    aa_metric_kernel<false><<<blocks, kThreads, 0, stream>>>(wh, n, anchors_dev, n_anchors, thr, part);
  YB_CHECK_CUDA(cudaGetLastError());
  aa_metric_fold_kernel<<<1, 32, 0, stream>>>(part, blocks, reinterpret_cast<long long*>(counts_dev), sums_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}

extern "C" size_t yb_kmeans_workspace_bytes(int64_t n_obs, int k, int trials) {
  if (n_obs <= 0 || k < 1 || trials < 1) return 0;
  return km_layout(n_obs, k, trials).total;
}

extern "C" int yb_kmeans(const double* obs_dev, int64_t n_obs, int k, int trials, const double* guess_dev,
                         double thresh, int check_every, double* books_dev, int32_t* sizes_dev, double* dist_dev,
                         int32_t* iters, void* workspace, size_t workspace_bytes, void* stream_) {
  YB_REQUIRE(obs_dev && guess_dev && books_dev && sizes_dev && dist_dev && iters && workspace,
             "kmeans: null argument");
  YB_REQUIRE(n_obs > 0 && n_obs < (int64_t(1) << 31), "kmeans: %lld observations", (long long)n_obs);
  YB_REQUIRE(k >= 1 && k <= YB_AA_MAX_ANCHORS && k <= n_obs, "kmeans: %d codes for %lld observations", k, (long long)n_obs);
  YB_REQUIRE(trials >= 1 && trials <= 65535 && check_every >= 1, "kmeans: %d trials, check every %d", trials,
             check_every);
  std::vector<SumNode> nodes;
  std::vector<int> ds;
  build_sum_tree(n_obs, nodes, ds);
  const KmLayout L = km_layout(n_obs, k, trials);
  YB_REQUIRE(workspace_bytes >= L.total, "kmeans: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  char* ws = static_cast<char*>(workspace);
  uint8_t* codes = reinterpret_cast<uint8_t*>(ws + L.codes);
  double* dist = reinterpret_cast<double*>(ws + L.dist);
  double* node_val = reinterpret_cast<double*>(ws + L.node_val);
  SumNode* d_nodes = reinterpret_cast<SumNode*>(ws + L.nodes);
  int* d_depth = reinterpret_cast<int*>(ws + L.depth);
  TrialState* st = reinterpret_cast<TrialState*>(ws + L.state);
  double* sums = reinterpret_cast<double*>(ws + L.sums);
  long long* counts = reinterpret_cast<long long*>(ws + L.counts);
  int* live = reinterpret_cast<int*>(ws + L.live);

  std::vector<TrialState> st0(trials, TrialState{kRun, k, 0, 0, HUGE_VAL});
  YB_CHECK_CUDA(cudaMemcpyAsync(d_nodes, nodes.data(), nodes.size() * sizeof(SumNode), cudaMemcpyHostToDevice, stream));
  YB_CHECK_CUDA(cudaMemcpyAsync(d_depth, ds.data(), ds.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
  YB_CHECK_CUDA(cudaMemcpyAsync(st, st0.data(), st0.size() * sizeof(TrialState), cudaMemcpyHostToDevice, stream));
  YB_CHECK_CUDA(cudaMemcpyAsync(live, &trials, sizeof(int), cudaMemcpyHostToDevice, stream));
  YB_CHECK_CUDA(cudaMemcpyAsync(books_dev, guess_dev, size_t(trials) * k * 2 * sizeof(double),
                                cudaMemcpyDeviceToDevice, stream));
  const dim3 vq_grid(unsigned(std::min<int64_t>((n_obs + kThreads - 1) / kThreads, 4 * num_sms())), unsigned(trials));
  const dim3 up_grid{unsigned(k), unsigned(trials)};
  const double2* obs = reinterpret_cast<const double2*>(obs_dev);
  // the loop has no host synchronisation but one read of the live-trial count every check_every iterations; a trial
  // that has finished makes every later launch return at once
  const int kMaxIter = 100000;
  int it = 0, left = trials;
  while (left > 0) {
    YB_REQUIRE(it < kMaxIter, "kmeans: no convergence after %d iterations", it);
    for (int q = 0; q < check_every; ++q, ++it) {
      km_vq_kernel<<<vq_grid, kThreads, 0, stream>>>(obs, n_obs, books_dev, k, st, codes, dist);
      km_mean_kernel<<<trials, kMeanThreads, 0, stream>>>(dist, n_obs, d_nodes, d_depth, L.depths, node_val, thresh,
                                                          st, dist_dev, live);
      km_update_kernel<<<up_grid, kThreads, 0, stream>>>(obs, n_obs, codes, k, st, sums, counts);
      km_compact_kernel<<<trials, 32, 0, stream>>>(sums, counts, k, st, books_dev);
    }
    YB_CHECK_CUDA(cudaGetLastError());
    YB_CHECK_CUDA(cudaMemcpyAsync(&left, live, sizeof(int), cudaMemcpyDeviceToHost, stream));
    YB_CHECK_CUDA(cudaStreamSynchronize(stream));
  }
  *iters = it;
  std::vector<TrialState> fin(trials);
  YB_CHECK_CUDA(cudaMemcpyAsync(fin.data(), st, fin.size() * sizeof(TrialState), cudaMemcpyDeviceToHost, stream));
  YB_CHECK_CUDA(cudaStreamSynchronize(stream));
  std::vector<int32_t> sizes(trials);
  for (int t = 0; t < trials; ++t) sizes[t] = fin[t].ncb;
  YB_CHECK_CUDA(cudaMemcpyAsync(sizes_dev, sizes.data(), sizes.size() * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  YB_CHECK_CUDA(cudaStreamSynchronize(stream));
  return YB_OK;
}

extern "C" int yb_anchor_evolve(const float* wh_dev, int64_t n, int n_anchors, const double* k0_dev,
                                const double* v_dev, int gen, double thr, int unit_exp, float* fit_dev,
                                uint8_t* accepted_dev, double* k_out_dev, void* workspace, size_t workspace_bytes,
                                void* stream_) {
  YB_REQUIRE(wh_dev && k0_dev && fit_dev && accepted_dev && k_out_dev && workspace && (v_dev || gen == 0),
             "anchor_evolve: null argument");
  YB_REQUIRE(n > 0 && n_anchors >= 1 && n_anchors <= YB_AA_MAX_ANCHORS && gen >= 0,
             "anchor_evolve: %lld labels, %d anchors, %d generations", (long long)n, n_anchors, gen);
  YB_REQUIRE(thr > 0.0 && thr < 1.0 && unit_exp < 0 && unit_exp > -200, "anchor_evolve: threshold %g, unit 2^%d", thr,
             unit_exp);
  // every term is at most 1 = 2^-unit_exp units: the sum of n terms must fit in 63 bits
  YB_REQUIRE(-unit_exp < 63 && n < (int64_t(1) << (63 + unit_exp)),
             "anchor_evolve: %lld labels overflow the exact sum at threshold %g", (long long)n, thr);
  YB_REQUIRE(workspace_bytes >= size_t(gen + 1) * sizeof(unsigned long long), "anchor_evolve: workspace of %zu bytes",
             workspace_bytes);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  unsigned long long* sums = static_cast<unsigned long long*>(workspace);
  YB_CHECK_CUDA(cudaMemsetAsync(sums, 0, size_t(gen + 1) * sizeof(unsigned long long), stream));
  YB_CHECK_CUDA(cudaMemsetAsync(accepted_dev, 0, size_t(gen > 0 ? gen : 1), stream));
  int per_sm = 0;
  YB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, aa_evolve_kernel, kThreads, 0));
  YB_REQUIRE(per_sm > 0, "anchor_evolve: the kernel cannot be resident");
  const int blocks = int(std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads,
                                                                int64_t(per_sm) * num_sms())));
  const float2* wh = reinterpret_cast<const float2*>(wh_dev);
  int64_t n_ = n;
  int na = n_anchors, gen_ = gen;
  float thr32 = float(thr);
  double unit = std::ldexp(1.0, unit_exp);
  void* args[] = {(void*)&wh, &n_, &na, (void*)&k0_dev, (void*)&v_dev, &gen_, &thr32, &unit, &sums, &fit_dev,
                  &accepted_dev, &k_out_dev};
  YB_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)aa_evolve_kernel, dim3(blocks), dim3(kThreads), args, 0, stream));
  return YB_OK;
}
