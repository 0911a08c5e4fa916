// The device parameter sampler of the training augmentations (Compose.apply_batch(..., generator=)).  One warp per
// image draws every random parameter of its transforms from Philox4x32-10 and carries the image's boxes through them;
// the result is the image's recipe in the yb_aug_image form yb_augment computes pixels from.  The rules (counters,
// words to numbers, fp32 operations and their order) are restated in oracle/sample_augment.py.
//
//   photometric  counter (i, t, 0, j) for block j = 0, 1, 2: words 0-6 the seven decisions, 7-10 the brightness,
//                contrast, saturation and hue factors, 11 the channel permutation
//   zoom-out     counter (i, t, 0, 0): apply, ratio, left, top
//   IoU crop     counter (i, t, round, 0xffffffff) word 0: the round's option; (i, t, round, trial): the trial's two
//                scales, left and top.  A round's trials are evaluated in parallel, one per lane, and the first
//                accepted trial in trial order wins
//   flip         counter (i, t, 0, 0) word 0
//
// Boxes live in the output rows of their image (global memory, read back through L1); the crop compacts them in
// order with a ballot.  Built with -fmad=false (Makefile) and written with _rn intrinsics: every product and sum is
// rounded on its own, as the host sampler's fp32 numpy / torch arithmetic rounds it.
#include "common.cuh"

namespace yb {
namespace {

constexpr int kWarps = 4;
constexpr uint32_t kFull = 0xffffffffu;

struct SampleArgs {
  yb_aug_sampler tr[YB_AUG_MAX_TRANSFORMS];
  int n_transforms;
};

__device__ __forceinline__ uint4 philox(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

__device__ __forceinline__ float uniform(uint32_t x) { return __fmul_rn(__uint2float_rn(x >> 8), 0x1p-24f); }
__device__ __forceinline__ int below(uint32_t x, int n) { return int((uint64_t(x) * uint32_t(n)) >> 32); }
__device__ __forceinline__ float from_range(const yb_aug_sampler& s, int j, uint32_t x) {
  return __fadd_rn(s.lo[j], __fmul_rn(uniform(x), s.span[j]));
}
__device__ __forceinline__ int trunc_mul(int a, float u) { return __float2int_rz(__fmul_rn(__int2float_rn(a), u)); }

struct Recipe {
  yb_aug_op* ops;
  int n, h, w;
  bool lane0;

  __device__ void push(int kind, int a0 = 0, int a1 = 0, int a2 = 0, int a3 = 0, int a4 = 0, int a5 = 0, int a6 = 0) {
    if (lane0) {
      yb_aug_op& op = ops[n];
      op.kind = kind;
      op.arg[0] = a0, op.arg[1] = a1, op.arg[2] = a2, op.arg[3] = a3, op.arg[4] = a4, op.arg[5] = a5, op.arg[6] = a6;
      op.factor = 0.0f;
      op.one_minus = 0.0f;
    }
    ++n;
  }
  __device__ void push_factor(int kind, float f) {
    push(kind, 0, kind == YB_AUG_CONTRAST ? h : 0, kind == YB_AUG_CONTRAST ? w : 0);
    if (lane0) {
      ops[n - 1].factor = f;
      ops[n - 1].one_minus = __double2float_rn(1.0 - double(f));   // torchvision's _blend: 1.0 - factor in double
    }
  }
};

__device__ void photometric(const yb_aug_sampler& s, uint4 c, uint2 key, Recipe& rc) {
  uint32_t x[12];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    c.w = uint32_t(j);
    const uint4 b = philox(c, key);
    x[4 * j] = b.x, x[4 * j + 1] = b.y, x[4 * j + 2] = b.z, x[4 * j + 3] = b.w;
  }
  float r[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) r[j] = uniform(x[j]);
  if (r[0] < s.p && (s.jitter & 1)) rc.push_factor(YB_AUG_BRIGHTNESS, from_range(s, 0, x[7]));
  const bool before = r[1] < 0.5f;
  if (before && r[2] < s.p && (s.jitter & 2)) rc.push_factor(YB_AUG_CONTRAST, from_range(s, 1, x[8]));
  if (r[3] < s.p && (s.jitter & 4)) rc.push_factor(YB_AUG_SATURATION, from_range(s, 2, x[9]));
  if (r[4] < s.p && (s.jitter & 8)) rc.push_factor(YB_AUG_HUE, from_range(s, 3, x[10]));
  if (!before && r[5] < s.p && (s.jitter & 2)) rc.push_factor(YB_AUG_CONTRAST, from_range(s, 1, x[8]));
  if (r[6] < s.p) {
    const int k = below(x[11], 6);                      // the permutations of (0, 1, 2) in lexicographic order
    const int a = k >> 1, b = (k & 1) ? (a == 2 ? 1 : 2) : (a == 0 ? 1 : 0);
    rc.push(YB_AUG_PERMUTE, a, b, 3 - a - b);
  }
}

// Boxes of rows [0, n) of `bx` / `lb`, processed by the warp's lanes.
__device__ void zoom_out(const yb_aug_sampler& s, uint4 c, uint2 key, Recipe& rc, float* bx, int n, int lane) {
  const uint4 x = philox(c, key);
  if (!(uniform(x.x) < s.p)) return;
  const float r = from_range(s, 0, x.y);
  const int cw = trunc_mul(rc.w, r), ch = trunc_mul(rc.h, r);
  const int left = trunc_mul(cw - rc.w, uniform(x.z)), top = trunc_mul(ch - rc.h, uniform(x.w));
  rc.push(YB_AUG_ZOOM_OUT, top, left, rc.h, rc.w, ch, cw, int(s.fill));
  rc.h = ch;
  rc.w = cw;
  const float fl = __int2float_rn(left), ft = __int2float_rn(top);
  for (int j = lane; j < n; j += 32) {
    float* b = bx + 4 * j;
    b[0] = __fadd_rn(b[0], fl), b[1] = __fadd_rn(b[1], ft), b[2] = __fadd_rn(b[2], fl), b[3] = __fadd_rn(b[3], ft);
  }
  __syncwarp();
}

__device__ void hflip(const yb_aug_sampler& s, uint4 c, uint2 key, Recipe& rc, float* bx, int n, int lane) {
  if (!(uniform(philox(c, key).x) < s.p)) return;
  rc.push(YB_AUG_HFLIP, rc.w);
  const float fw = __int2float_rn(rc.w);
  for (int j = lane; j < n; j += 32) {
    float* b = bx + 4 * j;
    const float x0 = b[0];
    b[0] = __fsub_rn(fw, b[2]);
    b[2] = __fsub_rn(fw, x0);
  }
  __syncwarp();
}

__device__ __forceinline__ bool centre_inside(const float* b, float l, float t, float r, float btm) {
  const float cx = __fmul_rn(0.5f, __fadd_rn(b[0], b[2])), cy = __fmul_rn(0.5f, __fadd_rn(b[1], b[3]));
  return l < cx && cx < r && t < cy && cy < btm;
}

// Returns the number of boxes kept.
__device__ int iou_crop(const yb_aug_sampler& s, uint4 c, uint2 key, Recipe& rc, float* bx, int64_t* lb, int n,
                        int lane, int32_t& status) {
  const float fw = __int2float_rn(rc.w), fh = __int2float_rn(rc.h);
  for (uint32_t round = 0; round < YB_AUG_CROP_ROUNDS; ++round) {
    c.z = round;
    c.w = 0xffffffffu;
    const double jac = s.options[below(philox(c, key).x, s.n_options)];
    if (jac >= 1.0) return n;                           // the image stays as it is
    for (int t0 = 0; t0 < s.trials; t0 += 32) {
      const int trial = t0 + lane;
      bool ok = false;
      int nw = 0, nh = 0, left = 0, top = 0;
      if (trial < s.trials) {
        c.w = uint32_t(trial);
        const uint4 x = philox(c, key);
        nw = __float2int_rz(__fmul_rn(fw, from_range(s, 0, x.x)));
        nh = __float2int_rz(__fmul_rn(fh, from_range(s, 0, x.y)));
        const double q = double(nw) / double(nh);       // the reference's Python division: inf / NaN fail the test
        left = trunc_mul(rc.w - nw, uniform(x.z));
        top = trunc_mul(rc.h - nh, uniform(x.w));
        ok = s.min_aspect <= q && q <= s.max_aspect && nw != 0 && nh != 0;
        if (ok) {
          const float l = __int2float_rn(left), t = __int2float_rn(top);
          const float r = __int2float_rn(left + nw), btm = __int2float_rn(top + nh);
          const float area2 = __fmul_rn(__fsub_rn(r, l), __fsub_rn(btm, t));
          bool any = false;
          float best = -INFINITY;
          for (int j = 0; j < n; ++j) {                 // torchvision's box_iou of the kept boxes with the window
            const float* b = bx + 4 * j;
            if (!centre_inside(b, l, t, r, btm)) continue;
            any = true;
            const float area1 = __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]));
            const float iw = fmaxf(__fsub_rn(fminf(b[2], r), fmaxf(b[0], l)), 0.0f);
            const float ih = fmaxf(__fsub_rn(fminf(b[3], btm), fmaxf(b[1], t)), 0.0f);
            const float inter = __fmul_rn(iw, ih);
            const float iou = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
            best = iou > best ? iou : best;
          }
          ok = any && !(double(best) < jac);
        }
      }
      const uint32_t acc = __ballot_sync(kFull, ok);
      if (!acc) continue;
      const int win = __ffs(acc) - 1;
      nw = __shfl_sync(kFull, nw, win);
      nh = __shfl_sync(kFull, nh, win);
      left = __shfl_sync(kFull, left, win);
      top = __shfl_sync(kFull, top, win);
      const float l = __int2float_rn(left), t = __int2float_rn(top);
      const float r = __int2float_rn(left + nw), btm = __int2float_rn(top + nh);
      const float cw = __int2float_rn(nw), ch = __int2float_rn(nh);
      int kept = 0;
      for (int j0 = 0; j0 < n; j0 += 32) {               // in-place compaction, order kept
        const int j = j0 + lane;
        float b[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        int64_t label = 0;
        bool in = false;
        if (j < n) {
          b[0] = bx[4 * j], b[1] = bx[4 * j + 1], b[2] = bx[4 * j + 2], b[3] = bx[4 * j + 3];
          label = lb[j];
          in = centre_inside(b, l, t, r, btm);
        }
        const uint32_t m = __ballot_sync(kFull, in);
        __syncwarp();                                   // every lane has read its row before any row is written
        if (in) {
          const int o = kept + __popc(m & ((1u << lane) - 1u));
          float* d = bx + 4 * o;
          d[0] = fminf(fmaxf(__fsub_rn(b[0], l), 0.0f), cw);
          d[1] = fminf(fmaxf(__fsub_rn(b[1], t), 0.0f), ch);
          d[2] = fminf(fmaxf(__fsub_rn(b[2], l), 0.0f), cw);
          d[3] = fminf(fmaxf(__fsub_rn(b[3], t), 0.0f), ch);
          lb[o] = label;
        }
        kept += __popc(m);
        __syncwarp();
      }
      rc.push(YB_AUG_CROP, top, left, nh, nw);
      rc.h = nh;
      rc.w = nw;
      return kept;
    }
  }
  status |= YB_AUG_ST_CROP_ROUNDS;
  return n;
}

__global__ void __launch_bounds__(32 * kWarps) augment_sample_kernel(
    const __grid_constant__ SampleArgs a, int n_images, const int64_t* __restrict__ key_dev,
    yb_aug_image* __restrict__ descs, const float* __restrict__ boxes, const int64_t* __restrict__ labels,
    const int32_t* __restrict__ box_start, float* boxes_out, int64_t* labels_out, int32_t* __restrict__ counts,
    int32_t* __restrict__ status) {
  const int img = int(blockIdx.x) * kWarps + int(threadIdx.x >> 5);
  const int lane = int(threadIdx.x & 31);
  if (img >= n_images) return;
  const uint2 key = make_uint2(uint32_t(key_dev[0]), uint32_t(key_dev[1]));
  yb_aug_image& d = descs[img];
  const int s = box_start[img];
  int n = box_start[img + 1] - s;
  float* bx = boxes_out + 4 * int64_t(s);
  int64_t* lb = labels_out + s;
  for (int j = lane; j < n; j += 32) {
#pragma unroll
    for (int k = 0; k < 4; ++k) bx[4 * j + k] = boxes[4 * (int64_t(s) + j) + k];
    lb[j] = labels[s + j];
  }
  __syncwarp();
  Recipe rc{d.ops, 0, d.src_h, d.src_w, lane == 0};
  int32_t st = 0;
  for (int t = 0; t < a.n_transforms; ++t) {
    const yb_aug_sampler& tr = a.tr[t];
    const uint4 c = make_uint4(uint32_t(img), uint32_t(t), 0u, 0u);
    switch (tr.kind) {
      case YB_AUG_S_PHOTOMETRIC:
        photometric(tr, c, key, rc);
        break;
      case YB_AUG_S_ZOOM_OUT:
        zoom_out(tr, c, key, rc, bx, n, lane);
        break;
      case YB_AUG_S_IOU_CROP:
        n = iou_crop(tr, c, key, rc, bx, lb, n, lane, st);
        break;
      case YB_AUG_S_HFLIP:
        hflip(tr, c, key, rc, bx, n, lane);
        break;
      default:
        break;
    }
  }
  if (lane == 0) {
    d.n_ops = rc.n;
    d.out_h = rc.h;
    d.out_w = rc.w;
    counts[img] = n;
    status[img] = st;
  }
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_augment_sample(int n_images, const yb_aug_sampler* transforms, int n_transforms,
                                 const int64_t* key_dev, yb_aug_image* descs_dev, const float* boxes_dev,
                                 const int64_t* labels_dev, const int32_t* box_start_dev, float* boxes_out_dev,
                                 int64_t* labels_out_dev, int32_t* counts_dev, int32_t* status_dev, void* stream_) {
  YB_REQUIRE(n_images > 0 && key_dev && descs_dev && box_start_dev && counts_dev && status_dev,
             "augment_sample: null argument or empty batch");
  YB_REQUIRE((boxes_dev == nullptr) == (labels_dev == nullptr) && (boxes_dev == nullptr) == (boxes_out_dev == nullptr) &&
                 (boxes_dev == nullptr) == (labels_out_dev == nullptr),
             "augment_sample: the box pointers are all set or all null");
  YB_REQUIRE(n_transforms >= 0 && n_transforms <= YB_AUG_MAX_TRANSFORMS && (n_transforms == 0 || transforms),
             "augment_sample: %d transforms (at most %d)", n_transforms, YB_AUG_MAX_TRANSFORMS);
  YB_REQUIRE(n_images <= (1 << 26), "augment_sample: %d images", n_images);
  SampleArgs a;
  memset(&a, 0, sizeof(a));
  a.n_transforms = n_transforms;
  int ops = 0, contrast = 0;
  for (int t = 0; t < n_transforms; ++t) {
    const yb_aug_sampler& s = transforms[t];
    switch (s.kind) {
      case YB_AUG_S_NONE:
        break;
      case YB_AUG_S_PHOTOMETRIC:
        YB_REQUIRE((s.jitter & ~15) == 0, "augment_sample: transform %d: jitter mask %d", t, s.jitter);
        ops += __builtin_popcount(unsigned(s.jitter)) + 1;
        contrast += (s.jitter >> 1) & 1;
        break;
      case YB_AUG_S_ZOOM_OUT:
        YB_REQUIRE((s.fill >> 24) == 0, "augment_sample: transform %d: fill %u", t, s.fill);
        ++ops;
        break;
      case YB_AUG_S_IOU_CROP:
        YB_REQUIRE(s.n_options > 0 && s.n_options <= YB_AUG_MAX_OPTIONS && s.trials >= 0,
                   "augment_sample: transform %d: %d options (1 to %d), %d trials", t, s.n_options, YB_AUG_MAX_OPTIONS,
                   s.trials);
        ++ops;
        break;
      case YB_AUG_S_HFLIP:
        ++ops;
        break;
      default:
        YB_REQUIRE(false, "augment_sample: transform %d has unknown kind %d", t, s.kind);
    }
    a.tr[t] = s;
  }
  YB_REQUIRE(ops <= YB_AUG_MAX_OPS && contrast <= YB_AUG_MAX_CONTRAST,
             "augment_sample: the transforms can draw %d ops (at most %d) and %d contrast ops (at most %d)", ops,
             YB_AUG_MAX_OPS, contrast, YB_AUG_MAX_CONTRAST);
  const unsigned blocks = unsigned((n_images + kWarps - 1) / kWarps);
  augment_sample_kernel<<<blocks, 32 * kWarps, 0, static_cast<cudaStream_t>(stream_)>>>(
      a, n_images, key_dev, descs_dev, boxes_dev, labels_dev, box_start_dev, boxes_out_dev, labels_out_dev, counts_dev,
      status_dev);
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
