// Baseline JPEG decode on the device, bit-identical to libjpeg's islow / fancy-upsampling / integer-YCbCr decode
// (the CPU decoder behind torchvision.io.decode_jpeg).  Host parser + five stages:
//   destuff   three launches: per-tile counts, a per-image scan, per-tile writes.  Removes the stuffed 0x00 after
//             0xFF, the fill 0xFFs and the RSTn markers, and records where each restart interval starts.
//   huffman   one cooperative launch (grid-wide barriers between phases).  Self-synchronising parallel decode
//             (Weissenberger & Schmidt, ICPP 2018 / arXiv:2111.09219): every image's destuffed bitstream is cut
//             into subsequences of kSubBits; each thread decodes its subsequence from an entry state (bit
//             position, block within the MCU, coefficient index) and records its exit state.  Round 0 guesses
//             the entry; round r takes the neighbour's exit of round r-1, until no exit changes (a fixed point is
//             the sequential decode, by induction from the known start).  A segmented scan of the per-
//             subsequence block counts and DC sums (reset at every restart) then places each subsequence's
//             blocks and DC predictors, and a last pass writes the coefficients.
//   idct      dequantise + islow IDCT per 8x8 block into per-component planes.
//   colour    fancy upsampling + YCbCr->RGB, written as HWC uint8.
#include <cooperative_groups.h>

#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace {

// Subsequence length of the parallel Huffman decode.  Measured on an H100 for 32 files of 640x480 4:2:0 (q75 / q95):
// 512 bits take 15 / 39 rounds and 1.23 / 3.09 ms in the Huffman kernel, 1024 bits 7 / 20 rounds and 1.10 / 2.66 ms,
// 2048 bits 3 / 9 rounds and 1.03 / 2.06 ms.  One 1280x720 file without DRI: 0.76, 0.85, 0.90 ms.
constexpr int kSubBits = 2048;
constexpr int kSubThreads = 128;    // subsequences per cooperative work item (one CTA)
constexpr int kTileBytes = 4096;    // destuff tile: 256 threads x 16 bytes
constexpr int kTileThreads = 256;
constexpr int32_t kTerminal = 0x7fffffff;   // exit position once the last MCU of an image has been decoded
constexpr int kMaxDstPerLaunch = 256;   // destination pointers per colour launch (kernel parameters)

__host__ __device__ inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }
__host__ __device__ inline int32_t cdiv(int64_t a, int64_t b) { return (int32_t)((a + b - 1) / b); }

struct SubState {
  int32_t pos;   // bit position in the image's destuffed stream (kTerminal: done)
  int32_t bz;    // block within the MCU << 8 | coefficient index (0 = the DC comes next)
};
struct SubAcc {
  int32_t blocks;   // blocks whose DC this subsequence decoded
  int32_t dc[3];    // DC differences since the last restart (or since the entry)
  int32_t reset;    // a restart happened inside
};

// Per-image record, computed identically on the host (launch sizes, workspace size) and on the device (setup
// kernel, from the copy of the infos inside src): the device never needs a second host-to-device copy.
struct ImgRec {
  int32_t W, H, ncomp, bpm, mcus_x, mcus_y, ri, n_int;
  int32_t scan_len, nsub, ntiles, nitems, blocks;
  int32_t hs[3], vs[3], hr[3], vr[3], dw[3], dh[3], pw[3], ph[3];
  uint8_t layout[10];    // block b of an MCU: component << 4 | v << 2 | h
  int64_t info_off, scan_src;                  // bytes into src
  int64_t meta, ds, ints, tiles, st0, st1, acc, pre, coef, plane[3];   // bytes into the workspace
  int64_t bytes;                                // workspace bytes of this image
  int32_t tile0, item0, blk0;                   // batch prefixes
  int64_t px0;
};

// meta words per image: [0] destuffed length, [1] intervals in use
__host__ __device__ inline void image_layout(const yb_jpeg_info& in, int64_t info_off, ImgRec& r) {
  r.W = in.width;
  r.H = in.height;
  r.ncomp = in.ncomp;
  r.bpm = in.blocks_per_mcu;
  r.mcus_x = in.mcus_x;
  r.mcus_y = in.mcus_y;
  r.ri = in.restart_interval;
  const int64_t mcus = (int64_t)in.mcus_x * in.mcus_y;
  r.n_int = r.ri ? cdiv(mcus, r.ri) : 1;
  r.scan_len = (int32_t)(in.scan_end - in.scan_begin);
  r.nsub = r.scan_len > 0 ? cdiv((int64_t)r.scan_len * 8, kSubBits) : 1;
  r.ntiles = r.scan_len > 0 ? cdiv(r.scan_len, kTileBytes) : 1;
  r.nitems = cdiv(r.nsub, kSubThreads);
  r.blocks = (int32_t)(mcus * r.bpm);
  int hmax = 1, vmax = 1;
  for (int c = 0; c < in.ncomp; ++c) {
    hmax = in.h_samp[c] > hmax ? in.h_samp[c] : hmax;
    vmax = in.v_samp[c] > vmax ? in.v_samp[c] : vmax;
  }
  int b = 0;
  for (int c = 0; c < 3; ++c) {
    const bool live = c < in.ncomp;
    const int h = live ? in.h_samp[c] : 1, v = live ? in.v_samp[c] : 1;
    r.hs[c] = in.ncomp == 1 ? 1 : h;      // a single-component scan is non-interleaved: one block per MCU
    r.vs[c] = in.ncomp == 1 ? 1 : v;
    r.hr[c] = hmax / h;
    r.vr[c] = vmax / v;
    r.dw[c] = cdiv((int64_t)in.width * h, hmax);
    r.dh[c] = cdiv((int64_t)in.height * v, vmax);
    r.pw[c] = live ? r.mcus_x * r.hs[c] * 8 : 0;
    r.ph[c] = live ? r.mcus_y * r.vs[c] * 8 : 0;
    if (live)
      for (int vv = 0; vv < r.vs[c]; ++vv)
        for (int hh = 0; hh < r.hs[c]; ++hh)
          if (b < 10) r.layout[b++] = (uint8_t)(c << 4 | vv << 2 | hh);
  }
  for (; b < 10; ++b) r.layout[b] = 0;
  r.info_off = info_off;
  r.scan_src = in.data_offset + in.scan_begin;
  int64_t o = 0;
  r.meta = o;   o += 64;
  r.ds = o;     o = align_up(o + r.scan_len + kSubBits / 8 + 64, 16);   // + readable slack past the last bit
  r.ints = o;   o = align_up(o + 4 * ((int64_t)r.n_int + 1), 16);
  r.tiles = o;  o = align_up(o + 8 * (int64_t)r.ntiles, 16);
  r.st0 = o;    o = align_up(o + 8 * (int64_t)r.nsub, 16);
  r.st1 = o;    o = align_up(o + 8 * (int64_t)r.nsub, 16);
  r.acc = o;    o = align_up(o + (int64_t)sizeof(SubAcc) * r.nsub, 16);
  r.pre = o;    o = align_up(o + (int64_t)sizeof(SubAcc) * r.nsub, 16);
  r.coef = o;   o = align_up(o + 128 * (int64_t)r.blocks, 256);
  for (int c = 0; c < 3; ++c) {
    r.plane[c] = o;
    o = align_up(o + (int64_t)r.pw[c] * r.ph[c], 256);
  }
  r.bytes = o;
}

struct BatchSize {
  int64_t bytes;    // workspace, records included
  int32_t tiles, items, blocks, max_nsub;
  int64_t px;
};

__host__ __device__ inline int64_t records_bytes(int n) { return align_up((int64_t)n * sizeof(ImgRec), 256) + 256; }   // + flags

BatchSize batch_size(int n, const yb_jpeg_info* infos) {
  BatchSize s{records_bytes(n), 0, 0, 0, 0, 0};
  for (int i = 0; i < n; ++i) {
    ImgRec r;
    image_layout(infos[i], 0, r);
    s.bytes += r.bytes;
    s.tiles += r.ntiles;
    s.items += r.nitems;
    s.blocks += r.blocks;
    s.max_nsub = std::max(s.max_nsub, r.nsub);
    s.px += (int64_t)r.W * r.H;
  }
  return s;
}

// ------------------------------------------------------------------------------------------------------------
// setup: one CTA computes every image's record and the batch prefixes (a block-wide scan per tile of images)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) jpeg_setup_kernel(int n, const uint8_t* __restrict__ src, uint8_t* ws) {
  ImgRec* recs = reinterpret_cast<ImgRec*>(ws);
  __shared__ int64_t s_bytes[1024], s_px[1024];
  __shared__ int32_t s_t[1024], s_i[1024], s_b[1024];
  __shared__ int64_t c_bytes, c_px;
  __shared__ int32_t c_t, c_i, c_b;
  if (threadIdx.x == 0) {
    c_bytes = records_bytes(n);
    c_px = 0;
    c_t = c_i = c_b = 0;
  }
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    ImgRec r;
    if (i < n) {
      const yb_jpeg_info& in = reinterpret_cast<const yb_jpeg_info*>(src)[i];
      image_layout(in, (int64_t)i * sizeof(yb_jpeg_info), r);
    } else {
      r.bytes = 0; r.ntiles = r.nitems = r.blocks = 0; r.W = r.H = 0;
    }
    s_bytes[threadIdx.x] = r.bytes;
    s_px[threadIdx.x] = (int64_t)r.W * r.H;
    s_t[threadIdx.x] = r.ntiles;
    s_i[threadIdx.x] = r.nitems;
    s_b[threadIdx.x] = r.blocks;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {    // inclusive Hillis-Steele scan
      int64_t a = 0, p = 0;
      int32_t t = 0, it = 0, bl = 0;
      if (threadIdx.x >= off) {
        a = s_bytes[threadIdx.x - off]; p = s_px[threadIdx.x - off];
        t = s_t[threadIdx.x - off]; it = s_i[threadIdx.x - off]; bl = s_b[threadIdx.x - off];
      }
      __syncthreads();
      s_bytes[threadIdx.x] += a; s_px[threadIdx.x] += p;
      s_t[threadIdx.x] += t; s_i[threadIdx.x] += it; s_b[threadIdx.x] += bl;
      __syncthreads();
    }
    if (i < n) {
      const int64_t base_bytes = c_bytes + s_bytes[threadIdx.x] - r.bytes;
      r.meta += base_bytes; r.ds += base_bytes; r.ints += base_bytes; r.tiles += base_bytes;
      r.st0 += base_bytes; r.st1 += base_bytes; r.acc += base_bytes; r.pre += base_bytes; r.coef += base_bytes;
      for (int c = 0; c < 3; ++c) r.plane[c] += base_bytes;
      r.tile0 = c_t + s_t[threadIdx.x] - r.ntiles;
      r.item0 = c_i + s_i[threadIdx.x] - r.nitems;
      r.blk0 = c_b + s_b[threadIdx.x] - r.blocks;
      r.px0 = c_px + s_px[threadIdx.x] - (int64_t)r.W * r.H;
      recs[i] = r;
    }
    __syncthreads();
    if (threadIdx.x == 1023) {
      c_bytes += s_bytes[1023]; c_px += s_px[1023]; c_t += s_t[1023]; c_i += s_i[1023]; c_b += s_b[1023];
    }
    __syncthreads();
  }
}

// index of the image whose [first, first + count) range of some per-batch numbering holds `idx`
template <typename F>
__device__ inline int find_image(const ImgRec* recs, int n, int64_t idx, F first) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first(recs[mid]) <= idx) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------------------
// destuff
// ------------------------------------------------------------------------------------------------------------
struct ByteClass {
  int emit;     // 1: contributes one data byte (b, or 0xFF for a stuffed FF 00 pair)
  int marker;   // 1: b is the 0xFF of an RSTn marker
  int bad;      // 1: the 0xFF of some other marker
  int code;     // the marker's second byte
};

__device__ inline ByteClass classify(const uint8_t* s, int len, int i) {
  const int b = s[i];
  const int prev = i > 0 ? s[i - 1] : 0;
  const int next = i + 1 < len ? s[i + 1] : 0;
  ByteClass c{0, 0, 0, next};
  if (b == 0xFF) {
    if (next == 0x00) c.emit = 1;
    else if (next >= 0xD0 && next <= 0xD7) c.marker = 1;
    else if (next != 0xFF) c.bad = 1;     // the host ends the segment at the first other marker: never expected
  } else if (prev != 0xFF) {
    c.emit = 1;
  }
  return c;
}

__global__ void __launch_bounds__(kTileThreads) jpeg_destuff_count_kernel(int n, const uint8_t* __restrict__ src,
                                                                          uint8_t* ws) {
  const ImgRec* recs = reinterpret_cast<const ImgRec*>(ws);
  const int img = find_image(recs, n, blockIdx.x, [](const ImgRec& r) { return (int64_t)r.tile0; });
  const ImgRec& r = recs[img];
  const int tile = blockIdx.x - r.tile0;
  const uint8_t* s = src + r.scan_src;
  int emit = 0, mark = 0;
  const int i0 = tile * kTileBytes + threadIdx.x * 16;
  for (int k = 0; k < 16; ++k) {
    const int i = i0 + k;
    if (i < r.scan_len) {
      const ByteClass c = classify(s, r.scan_len, i);
      emit += c.emit;
      mark += c.marker;
    }
  }
  __shared__ int se[kTileThreads / 32], sm[kTileThreads / 32];
  for (int o = 16; o; o >>= 1) {
    emit += __shfl_xor_sync(0xffffffffu, emit, o);
    mark += __shfl_xor_sync(0xffffffffu, mark, o);
  }
  if ((threadIdx.x & 31) == 0) { se[threadIdx.x >> 5] = emit; sm[threadIdx.x >> 5] = mark; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, m = 0;
    for (int w = 0; w < kTileThreads / 32; ++w) { a += se[w]; m += sm[w]; }
    int32_t* t = reinterpret_cast<int32_t*>(ws + r.tiles) + 2 * tile;
    t[0] = a;
    t[1] = m;
  }
}

__global__ void __launch_bounds__(32) jpeg_destuff_scan_kernel(int n, uint8_t* ws, int32_t* status) {
  const ImgRec* recs = reinterpret_cast<const ImgRec*>(ws);
  const ImgRec& r = recs[blockIdx.x];
  int32_t* t = reinterpret_cast<int32_t*>(ws + r.tiles);
  int carry_e = 0, carry_m = 0;
  for (int base = 0; base < r.ntiles; base += 32) {
    const int k = base + threadIdx.x;
    int e = k < r.ntiles ? t[2 * k] : 0, m = k < r.ntiles ? t[2 * k + 1] : 0;
    int ie = e, im = m;
    for (int o = 1; o < 32; o <<= 1) {
      const int pe = __shfl_up_sync(0xffffffffu, ie, o), pm = __shfl_up_sync(0xffffffffu, im, o);
      if ((int)threadIdx.x >= o) { ie += pe; im += pm; }
    }
    if (k < r.ntiles) { t[2 * k] = carry_e + ie - e; t[2 * k + 1] = carry_m + im - m; }
    carry_e += __shfl_sync(0xffffffffu, ie, 31);
    carry_m += __shfl_sync(0xffffffffu, im, 31);
  }
  if (threadIdx.x == 0) {
    int32_t* meta = reinterpret_cast<int32_t*>(ws + r.meta);
    int32_t* ints = reinterpret_cast<int32_t*>(ws + r.ints);
    const int used = min(carry_m, r.n_int - 1) + 1;
    meta[0] = carry_e;
    meta[1] = used;
    ints[0] = 0;
    ints[used] = carry_e;
    if (carry_m != r.n_int - 1) atomicOr(status + blockIdx.x, YB_JPEG_ST_RESTART);
  }
  uint8_t* ds = ws + r.ds;
  for (int k = carry_e + threadIdx.x; k < carry_e + 16; k += 32) ds[k] = 0xFF;   // readable padding
}

__global__ void __launch_bounds__(kTileThreads) jpeg_destuff_write_kernel(int n, const uint8_t* __restrict__ src,
                                                                          uint8_t* ws, int32_t* status) {
  const ImgRec* recs = reinterpret_cast<const ImgRec*>(ws);
  const int img = find_image(recs, n, blockIdx.x, [](const ImgRec& r) { return (int64_t)r.tile0; });
  const ImgRec& r = recs[img];
  const int tile = blockIdx.x - r.tile0;
  const uint8_t* s = src + r.scan_src;
  const int32_t* t = reinterpret_cast<const int32_t*>(ws + r.tiles) + 2 * tile;
  uint8_t* ds = ws + r.ds;
  int32_t* ints = reinterpret_cast<int32_t*>(ws + r.ints);
  const int used = reinterpret_cast<const int32_t*>(ws + r.meta)[1];
  const int i0 = tile * kTileBytes + threadIdx.x * 16;
  int emit = 0, mark = 0, bad = 0;
  ByteClass cls[16];
  for (int k = 0; k < 16; ++k) {
    const int i = i0 + k;
    cls[k] = i < r.scan_len ? classify(s, r.scan_len, i) : ByteClass{0, 0, 0, 0};
    emit += cls[k].emit;
    mark += cls[k].marker;
    bad |= cls[k].bad;
  }
  __shared__ int se[kTileThreads], sm[kTileThreads];
  se[threadIdx.x] = emit;
  sm[threadIdx.x] = mark;
  __syncthreads();
  for (int o = 1; o < kTileThreads; o <<= 1) {
    const int a = threadIdx.x >= o ? se[threadIdx.x - o] : 0, m = threadIdx.x >= o ? sm[threadIdx.x - o] : 0;
    __syncthreads();
    se[threadIdx.x] += a;
    sm[threadIdx.x] += m;
    __syncthreads();
  }
  int out = t[0] + se[threadIdx.x] - emit;
  int mk = t[1] + sm[threadIdx.x] - mark;
  for (int k = 0; k < 16; ++k) {
    if (cls[k].emit) ds[out++] = s[i0 + k];      // a stuffed pair emits its 0xFF
    if (cls[k].marker) {
      if (cls[k].code != 0xD0 + (mk & 7)) bad = 1;
      if (mk + 1 < used) ints[mk + 1] = out;
      ++mk;
    }
  }
  if (bad) atomicOr(status + img, YB_JPEG_ST_RESTART);
}

// ------------------------------------------------------------------------------------------------------------
// Huffman
// ------------------------------------------------------------------------------------------------------------
__constant__ uint8_t kZigzag[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};


constexpr int kLutBits = 9;

// Canonical Huffman tables of one image in shared memory, libjpeg's derived form (maxcode / valoffset per length)
// plus a 9-bit lookup table for the short codes.  Slot t = component * 2 + (0: DC, 1: AC).
struct HuffSmem {
  uint16_t lut[6][1 << kLutBits];   // len << 8 | symbol for codes of <= 9 bits, 0 = longer code or none
  int32_t maxcode[6][17];           // largest code of each length, -1 if none
  int32_t valoff[6][17];            // symbol index = code + valoff
  uint8_t vals[6][256];
  uint8_t layout[10];
  int32_t img;
};

__device__ void load_tables(HuffSmem& T, const yb_jpeg_info& in, const ImgRec& r, int img) {
  if (T.img == img) return;    // uniform over the CTA: every thread read the same T.img after a barrier
  __syncthreads();
  if (threadIdx.x < 6) {
    const int t = threadIdx.x, c = t >> 1, ac = t & 1;
    if (c < in.ncomp) {
      const uint8_t* bits = ac ? in.ac_bits[c] : in.dc_bits[c];
      int code = 0, k = 0;
      for (int l = 1; l <= 16; ++l) {
        const int cnt = bits[l - 1];
        T.maxcode[t][l] = cnt ? code + cnt - 1 : -1;
        T.valoff[t][l] = k - code;
        k += cnt;
        code = (code + cnt) << 1;
      }
      for (int v = 0; v < 256; ++v) T.vals[t][v] = v < k ? (ac ? in.ac_vals[c][v] : in.dc_vals[c][v & 15]) : 0;
    }
  }
  if (threadIdx.x < 10) T.layout[threadIdx.x] = r.layout[threadIdx.x];
  __syncthreads();
  for (int e = threadIdx.x; e < 6 * (1 << kLutBits); e += blockDim.x) {
    const int t = e >> kLutBits, x = e & ((1 << kLutBits) - 1);
    uint16_t v = 0;
    if ((t >> 1) < in.ncomp) {
      for (int l = 1; l <= kLutBits; ++l) {
        const int code = x >> (kLutBits - l);
        if (code <= T.maxcode[t][l]) {    // canonical codes: lengths in increasing order, as libjpeg's decoder
          v = (uint16_t)(l << 8 | T.vals[t][(code + T.valoff[t][l]) & 255]);
          break;
        }
      }
    }
    T.lut[t][x] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) T.img = img;
  __syncthreads();
}

// A window of three big-endian words of the destuffed stream, held in registers: a symbol reads one word from memory
// every 32 bits it consumes, one word ahead of need (the buffer has readable slack past its end).
struct Bits {
  const uint32_t* w;
  uint32_t w0, w1, w2;
  int32_t wi;   // index of w0

  __device__ static uint32_t be(uint32_t x) { return __byte_perm(x, 0, 0x0123); }
  __device__ void seek(int32_t pos) {
    wi = pos >> 5;
    w0 = be(w[wi]);
    w1 = be(w[wi + 1]);
    w2 = be(w[wi + 2]);
  }
  __device__ void advance(int32_t pos) {   // pos moved forward by at most 32 bits since the last call
    if ((pos >> 5) > wi) {
      w0 = w1;
      w1 = w2;
      w2 = be(w[wi + 3]);
      ++wi;
    }
  }
  __device__ uint32_t peek(int32_t pos) const { return __funnelshift_l(w1, w0, pos & 31); }   // 32 bits at pos
};

struct Dec {
  int32_t pos, b, z, r;   // bit position, block within the MCU, coefficient index, restart interval
  uint32_t dc[3];         // DC predictor (write pass) or DC differences since the entry / last restart
  int32_t blocks;         // blocks whose DC has been decoded (write pass: from the start of the image)
  int32_t reset, bad;
};

__device__ inline int find_interval(const int32_t* ints, int used, int32_t pos) {
  int lo = 0, hi = used - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ints[mid] * 8 <= pos) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct Geo {
  int32_t bpm, blocks, ri;   // blocks per MCU, blocks of the image, MCUs per restart interval
};

// Decodes symbols from state `d` until the first symbol boundary at or past bit `end` (or the end of the image).
// The same code serves the synchronisation rounds (kWrite = false: only the state and the counts) and the final
// pass (kWrite: coefficients, and every check of the status bits; those paths start from correct states).
template <bool kWrite>
__device__ inline void decode_until(const HuffSmem& T, const uint32_t* words, const int32_t* ints, int used,
                                    const Geo g, Dec& d, int32_t end, int16_t* coef) {
  int32_t pos = d.pos, b = d.b, z = d.z, r = d.r, blocks = d.blocks, bad = 0, reset = 0;
  uint32_t dc0 = d.dc[0], dc1 = d.dc[1], dc2 = d.dc[2];
  int16_t* blk = nullptr;
  if (kWrite && z != 0 && blocks >= 1 && blocks <= g.blocks) blk = coef + (int64_t)(blocks - 1) * 64;
  Bits br;
  br.w = words;
  br.seek(pos);
  int32_t E = ints[r + 1] * 8;
  while (pos < end) {
    const uint32_t bits = br.peek(pos);
    const int c = T.layout[b] >> 4;
    const int t = c * 2 + (z ? 1 : 0);
    const uint32_t e = T.lut[t][bits >> (32 - kLutBits)];
    int len, sym;
    if (e) {
      len = e >> 8;
      sym = e & 255;
    } else {
      len = 0;
      sym = 0;
      for (int l = kLutBits + 1; l <= 16; ++l) {
        const int code = (int)(bits >> (32 - l));
        if (code <= T.maxcode[t][l]) {
          len = l;
          sym = T.vals[t][(code + T.valoff[t][l]) & 255];
          break;
        }
      }
      if (!len) {
        len = 16;
        bad |= YB_JPEG_ST_HUFFMAN;
      }
    }
    const int s = sym & 15;
    int32_t v = 0;
    if (s) {
      const uint32_t x = (bits << len) >> (32 - s);    // len + s <= 32: the extra bits are in the same window
      v = (int32_t)x - ((x >> (s - 1)) ? 0 : (1 << s) - 1);    // HUFF_EXTEND
    }
    pos += len + s;
    br.advance(pos);
    if (z == 0) {               // DC difference (the parser allows categories 0..11 only)
      const uint32_t p = (c == 0 ? dc0 += (uint32_t)v : c == 1 ? dc1 += (uint32_t)v : dc2 += (uint32_t)v);
      if (kWrite) {
        if (blocks < g.blocks) {
          blk = coef + (int64_t)blocks * 64;
          blk[0] = (int16_t)p;    // libjpeg keeps the int predictor and stores a JCOEF
        } else {
          blk = nullptr;
          bad |= YB_JPEG_ST_TRUNCATED;
        }
      }
      blocks++;
      z = 1;
    } else {
      const int run = sym >> 4;
      if (s) {
        z += run;
        if (z > 63) {
          bad |= YB_JPEG_ST_COEF;
          z = 63;
        }
        if (kWrite && blk) blk[kZigzag[z]] = (int16_t)v;
        z++;
      } else if (run == 15) {   // ZRL
        z += 16;
        if (z > 64) {
          bad |= YB_JPEG_ST_COEF;
          z = 64;
        }
      } else {                  // EOB
        z = 64;
      }
      if (z == 64) {
        z = 0;
        if (++b == g.bpm) b = 0;
      }
    }
    // End of a restart interval: fewer than 8 bits left and all of them 1s (the encoder's padding; no code of an
    // accepted table is all 1s, so a pending code cannot look like padding).  The state then becomes the next
    // interval's start, the same for every path that gets here: restarts are free synchronisation points.
    if (pos >= E - 7) {
      const int rem = E - pos;
      if (rem <= 0 || (br.peek(pos) >> (32 - rem)) == (1u << rem) - 1u) {
        if (rem < 0 || b || z) bad |= YB_JPEG_ST_TRUNCATED;
        r++;
        b = z = 0;
        dc0 = dc1 = dc2 = 0;
        reset = 1;
        blk = nullptr;
        if (r >= used) {
          pos = kTerminal;
          break;
        }
        pos = ints[r] * 8;
        E = ints[r + 1] * 8;
        br.seek(pos);
        if (kWrite && (int64_t)blocks != (int64_t)r * g.ri * g.bpm) bad |= YB_JPEG_ST_TRUNCATED;
      }
    }
  }
  d.pos = pos;
  d.b = b;
  d.z = z;
  d.r = r;
  d.blocks = blocks;
  d.dc[0] = dc0;
  d.dc[1] = dc1;
  d.dc[2] = dc2;
  d.reset |= reset;
  d.bad |= bad;
}

struct ImgView {
  const uint32_t* words;
  const int32_t* ints;
  int32_t ds_bits, used;
  SubState* st0;
  SubState* st1;
  SubAcc* acc;
  SubAcc* pre;
  int16_t* coef;
};

__device__ inline ImgView view(uint8_t* ws, const ImgRec& R) {
  const int32_t* meta = reinterpret_cast<const int32_t*>(ws + R.meta);
  ImgView v;
  v.words = reinterpret_cast<const uint32_t*>(ws + R.ds);
  v.ints = reinterpret_cast<const int32_t*>(ws + R.ints);
  v.ds_bits = meta[0] * 8;
  v.used = meta[1];
  v.st0 = reinterpret_cast<SubState*>(ws + R.st0);
  v.st1 = reinterpret_cast<SubState*>(ws + R.st1);
  v.acc = reinterpret_cast<SubAcc*>(ws + R.acc);
  v.pre = reinterpret_cast<SubAcc*>(ws + R.pre);
  v.coef = reinterpret_cast<int16_t*>(ws + R.coef);
  return v;
}

__device__ inline void start(Dec& d, const ImgView& v, SubState e) {
  d.pos = e.pos >= v.ds_bits ? kTerminal : e.pos;
  d.b = e.bz >> 8;
  d.z = e.bz & 255;
  d.r = d.pos == kTerminal ? 0 : find_interval(v.ints, v.used, d.pos);
  d.reset = d.bad = 0;
}

__device__ inline SubAcc combine(const SubAcc& a, const SubAcc& b) {
  SubAcc o;
  o.blocks = a.blocks + b.blocks;
  for (int c = 0; c < 3; ++c) o.dc[c] = b.reset ? b.dc[c] : (int32_t)((uint32_t)a.dc[c] + (uint32_t)b.dc[c]);
  o.reset = a.reset | b.reset;
  return o;
}

__global__ void __launch_bounds__(kSubThreads) jpeg_huffman_kernel(int n, int total_items, int max_rounds,
                                                                    const uint8_t* __restrict__ src, uint8_t* ws,
                                                                    int32_t* status) {
  cg::grid_group grid = cg::this_grid();
  const ImgRec* recs = reinterpret_cast<const ImgRec*>(ws);
  volatile int32_t* flags = reinterpret_cast<volatile int32_t*>(ws + records_bytes(n) - 256);
  __shared__ HuffSmem T;
  __shared__ SubAcc scan[kSubThreads];
  if (threadIdx.x == 0) T.img = -1;
  __syncthreads();
  auto item_first = [](const ImgRec& r) { return (int64_t)r.item0; };

  // 1. synchronisation rounds
  int round = 0;
  for (;; ++round) {
    if (blockIdx.x == 0 && threadIdx.x == 0) flags[(round + 1) % 3] = 0;
    bool changed = false;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const int img = find_image(recs, n, item, item_first);
      const ImgRec& R = recs[img];
      load_tables(T, *reinterpret_cast<const yb_jpeg_info*>(src + R.info_off), R, img);
      const int j = (item - R.item0) * kSubThreads + threadIdx.x;
      if (j >= R.nsub) continue;
      const ImgView v = view(ws, R);
      SubState entry{0, 0};
      SubState* prev = (round & 1) ? v.st0 : v.st1;
      SubState* cur = (round & 1) ? v.st1 : v.st0;
      if (j > 0) entry = round == 0 ? SubState{j * kSubBits, 0} : prev[j - 1];
      Dec d;
      start(d, v, entry);
      d.dc[0] = d.dc[1] = d.dc[2] = 0;
      d.blocks = 0;
      if (d.pos != kTerminal)
        decode_until<false>(T, v.words, v.ints, v.used, Geo{R.bpm, R.blocks, R.ri}, d, (j + 1) * kSubBits, nullptr);
      const SubState out{d.pos, d.b << 8 | d.z};
      if (round > 0) {
        const SubState old = prev[j];
        changed |= old.pos != out.pos || old.bz != out.bz;
      }
      cur[j] = out;
      v.acc[j] = SubAcc{d.blocks, {(int32_t)d.dc[0], (int32_t)d.dc[1], (int32_t)d.dc[2]}, d.reset};
    }
    if (changed) flags[round % 3] = 1;
    grid.sync();
    if (round > 0 && flags[round % 3] == 0) break;
    if (round >= max_rounds) {     // cannot happen (round nsub is always a fixed point); fail safe, never hang
      for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        atomicOr(status + i, YB_JPEG_ST_TRUNCATED);
      break;
    }
  }
  const int fin = round & 1;

  // 2. per image: segmented exclusive scan of (blocks, DC sums) over the subsequences
  for (int img = blockIdx.x; img < n; img += gridDim.x) {
    const ImgRec& R = recs[img];
    const ImgView v = view(ws, R);
    SubAcc carry{0, {0, 0, 0}, 0};
    for (int base = 0; base < R.nsub; base += kSubThreads) {
      const int j = base + threadIdx.x;
      const SubAcc x = j < R.nsub ? v.acc[j] : SubAcc{0, {0, 0, 0}, 0};
      scan[threadIdx.x] = x;
      __syncthreads();
      for (int o = 1; o < kSubThreads; o <<= 1) {
        SubAcc y = scan[threadIdx.x];
        if ((int)threadIdx.x >= o) y = combine(scan[threadIdx.x - o], y);
        __syncthreads();
        scan[threadIdx.x] = y;
        __syncthreads();
      }
      if (j < R.nsub) v.pre[j] = threadIdx.x ? combine(carry, scan[threadIdx.x - 1]) : carry;
      const SubAcc tile = scan[kSubThreads - 1];
      __syncthreads();
      carry = combine(carry, tile);
    }
    if (threadIdx.x == 0) {
      const SubState last = (fin ? v.st1 : v.st0)[R.nsub - 1];
      if (carry.blocks != R.blocks || last.pos != kTerminal) atomicOr(status + img, YB_JPEG_ST_TRUNCATED);
    }
  }
  grid.sync();

  // 3. coefficients, from the converged entry states
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int img = find_image(recs, n, item, item_first);
    const ImgRec& R = recs[img];
    load_tables(T, *reinterpret_cast<const yb_jpeg_info*>(src + R.info_off), R, img);
    const int j = (item - R.item0) * kSubThreads + threadIdx.x;
    if (j >= R.nsub) continue;
    const ImgView v = view(ws, R);
    const SubState entry = j > 0 ? (fin ? v.st1 : v.st0)[j - 1] : SubState{0, 0};
    Dec d;
    start(d, v, entry);
    const SubAcc p = v.pre[j];
    d.dc[0] = p.dc[0];
    d.dc[1] = p.dc[1];
    d.dc[2] = p.dc[2];
    d.blocks = p.blocks;
    if (d.pos != kTerminal)
      decode_until<true>(T, v.words, v.ints, v.used, Geo{R.bpm, R.blocks, R.ri}, d, (j + 1) * kSubBits, v.coef);
    if (d.bad) atomicOr(status + img, d.bad);
  }
}

// ------------------------------------------------------------------------------------------------------------
// dequantise + islow IDCT (libjpeg's jpeg_idct_islow: 13-bit constants, PASS1_BITS = 2, 64-bit products)
// ------------------------------------------------------------------------------------------------------------
__device__ inline void idct8(const int64_t* x, int64_t* out, int shift) {
  const int64_t z2 = x[2], z3 = x[6];
  const int64_t z1 = (z2 + z3) * 4433;
  const int64_t tmp2 = z1 - z3 * 15137, tmp3 = z1 + z2 * 6270;
  const int64_t tmp0 = (x[0] + x[4]) * 8192, tmp1 = (x[0] - x[4]) * 8192;
  const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int64_t o0 = x[7], o1 = x[5], o2 = x[3], o3 = x[1];
  int64_t a1 = o0 + o3, a2 = o1 + o2, a3 = o0 + o2, a4 = o1 + o3;
  const int64_t z5 = (a3 + a4) * 9633;
  o0 *= 2446; o1 *= 16819; o2 *= 25172; o3 *= 12299;
  a1 *= -7373; a2 *= -20995;
  a3 = a3 * -16069 + z5;
  a4 = a4 * -3196 + z5;
  o0 += a1 + a3; o1 += a2 + a4; o2 += a2 + a3; o3 += a1 + a4;
  const int64_t r = (int64_t)1 << (shift - 1);
  out[0] = (t10 + o3 + r) >> shift; out[7] = (t10 - o3 + r) >> shift;
  out[1] = (t11 + o2 + r) >> shift; out[6] = (t11 - o2 + r) >> shift;
  out[2] = (t12 + o1 + r) >> shift; out[5] = (t12 - o1 + r) >> shift;
  out[3] = (t13 + o0 + r) >> shift; out[4] = (t13 - o0 + r) >> shift;
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(int n, int total_blocks, const uint8_t* __restrict__ src,
                                                         uint8_t* ws, int32_t* status) {
  const int gb = blockIdx.x * blockDim.x + threadIdx.x;
  if (gb >= total_blocks) return;
  const ImgRec* recs = reinterpret_cast<const ImgRec*>(ws);
  const int img = find_image(recs, n, gb, [](const ImgRec& r) { return (int64_t)r.blk0; });
  const ImgRec& R = recs[img];
  const int g = gb - R.blk0;
  const int m = g / R.bpm, lay = R.layout[g % R.bpm];
  const int c = lay >> 4;
  const int by = (m / R.mcus_x) * R.vs[c] + ((lay >> 2) & 3), bx = (m % R.mcus_x) * R.hs[c] + (lay & 3);
  const uint16_t* q = reinterpret_cast<const yb_jpeg_info*>(src + R.info_off)->quant[c];
  const int4* cp = reinterpret_cast<const int4*>(ws + R.coef + (int64_t)g * 128);
  int64_t blk[64];
  bool bad = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int4 w = cp[k];
    const int32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int i = k * 8 + 2 * h;
      blk[i] = (int64_t)(int16_t)(words[h] & 0xffff) * q[i];
      blk[i + 1] = (int64_t)(int16_t)((uint32_t)words[h] >> 16) * q[i + 1];
    }
  }
#pragma unroll
  for (int i = 0; i < 64; ++i) bad |= blk[i] > 32767 || blk[i] < -32767;   // libjpeg's SIMD multiplies in 16 bits
  int64_t col[8], res[8];
#pragma unroll
  for (int x = 0; x < 8; ++x) {       // pass 1: columns
#pragma unroll
    for (int y = 0; y < 8; ++y) col[y] = blk[y * 8 + x];
    idct8(col, res, 11);
#pragma unroll
    for (int y = 0; y < 8; ++y) {
      blk[y * 8 + x] = res[y];
      bad |= res[y] > 32767 || res[y] < -32768;   // and keeps pass 1 in 16 bits
    }
  }
  uint8_t* out = ws + R.plane[c] + (int64_t)by * 8 * R.pw[c] + bx * 8;
#pragma unroll
  for (int y = 0; y < 8; ++y) {       // pass 2: rows
    idct8(blk + y * 8, res, 18);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      bad |= res[x] < -512 || res[x] > 511;   // where C's range_limit[x & 1023] and SIMD saturation agree
      const uint32_t p = (uint32_t)min(max(res[x] + 128, (int64_t)0), (int64_t)255);
      if (x < 4) lo |= p << (8 * x); else hi |= p << (8 * (x - 4));
    }
    *reinterpret_cast<uint2*>(out + (int64_t)y * R.pw[c]) = make_uint2(lo, hi);
  }
  if (bad) atomicOr(status + img, YB_JPEG_ST_RANGE);
}

// ------------------------------------------------------------------------------------------------------------
// fancy upsampling + YCbCr -> RGB (libjpeg's jdsample.c / jdcolor.c integer arithmetic)
// ------------------------------------------------------------------------------------------------------------
struct DstPtrs {
  uint8_t* dst[kMaxDstPerLaunch];
};

// Component sample at output pixel (x, y): fullsize; h2v1 fancy (3a + neighbour + 1 | 2) >> 2; h2v2 fancy
// (3 * (3a + a_v) + (3b + b_v) + 8 | 7) >> 4; neighbours replicated at the downsampled width / height.  libjpeg
// takes the fancy filters only when the downsampled width exceeds 2, else it replicates each sample.
__device__ inline int comp_sample(const uint8_t* P, int pw, int dw, int dh, int hr, int vr, int x, int y) {
  if (hr == 1 && vr == 1) return P[(int64_t)y * pw + x];
  const int i = x >> 1;
  const int yy = vr == 2 ? y >> 1 : y;
  if (dw <= 2) return P[(int64_t)yy * pw + i];
  const int odd = x & 1;
  const int i2 = odd ? min(i + 1, dw - 1) : max(i - 1, 0);
  if (vr == 1) {
    const uint8_t* row = P + (int64_t)y * pw;
    return (3 * row[i] + row[i2] + 1 + odd) >> 2;
  }
  const int y2 = (y & 1) ? min(yy + 1, dh - 1) : max(yy - 1, 0);
  const uint8_t* r0 = P + (int64_t)yy * pw;
  const uint8_t* r1 = P + (int64_t)y2 * pw;
  const int a = 3 * r0[i] + r1[i], b = 3 * r0[i2] + r1[i2];
  return (3 * a + b + 8 - odd) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(int n, int first, int count, int64_t px_begin,
                                                          int64_t px_end, uint8_t* ws,
                                                          const __grid_constant__ DstPtrs dst) {
  const ImgRec* recs = reinterpret_cast<const ImgRec*>(ws) + first;
  for (int64_t p = px_begin + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < px_end;
       p += (int64_t)gridDim.x * blockDim.x) {
    const int k = find_image(recs, count, p, [](const ImgRec& r) { return r.px0; });
    const ImgRec& R = recs[k];
    const int64_t q = p - R.px0;
    const int y = (int)(q / R.W), x = (int)(q - (int64_t)y * R.W);
    int rgb[3];
    const int Y = comp_sample(ws + R.plane[0], R.pw[0], R.dw[0], R.dh[0], R.hr[0], R.vr[0], x, y);
    if (R.ncomp == 1) {
      rgb[0] = rgb[1] = rgb[2] = Y;
    } else {
      const int cb = comp_sample(ws + R.plane[1], R.pw[1], R.dw[1], R.dh[1], R.hr[1], R.vr[1], x, y) - 128;
      const int cr = comp_sample(ws + R.plane[2], R.pw[2], R.dw[2], R.dh[2], R.hr[2], R.vr[2], x, y) - 128;
      rgb[0] = Y + ((91881 * cr + 32768) >> 16);                 // FIX(1.40200)
      rgb[1] = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);   // FIX(0.34414), FIX(0.71414)
      rgb[2] = Y + ((116130 * cb + 32768) >> 16);                // FIX(1.77200)
    }
    uint8_t* o = dst.dst[k] + q * 3;
    o[0] = (uint8_t)min(max(rgb[0], 0), 255);
    o[1] = (uint8_t)min(max(rgb[1], 0), 255);
    o[2] = (uint8_t)min(max(rgb[2], 0), 255);
  }
}

// ------------------------------------------------------------------------------------------------------------
// host parser
// ------------------------------------------------------------------------------------------------------------
const uint8_t kZigzagHost[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

constexpr int64_t kMaxScanBytes = (int64_t)1 << 27;     // bit positions stay in int32
constexpr int64_t kMaxPixels = (int64_t)1 << 28;

int unsupported(yb_jpeg_info* o, const char* fmt, int a = 0) {
  o->supported = 0;
  snprintf(o->reason, sizeof(o->reason), fmt, a);
  return YB_OK;
}

struct HuffTable {
  bool set = false;
  uint8_t bits[16];
  uint8_t vals[256];
  int nvals = 0;
};

}  // namespace

extern "C" int yb_jpeg_parse(const uint8_t* d, int64_t len, yb_jpeg_info* o) {
  YB_REQUIRE(o != nullptr && (d != nullptr || len == 0) && len >= 0, "yb_jpeg_parse: null arguments");
  memset(o, 0, sizeof(*o));
  if (len < 4 || d[0] != 0xFF || d[1] != 0xD8) return unsupported(o, "not a JPEG file (no SOI marker)");
  HuffTable ht[2][4];
  uint16_t qt[4][64];
  bool qset[4] = {false, false, false, false};
  bool have_sof = false, jfif = false, adobe = false;
  int adobe_transform = -1;
  int ids[3] = {0, 0, 0}, tq[3] = {0, 0, 0}, hs[3] = {0, 0, 0}, vs[3] = {0, 0, 0};
  int nf = 0, W = 0, H = 0;
  int64_t i = 2;
  for (;;) {
    if (i >= len || d[i] != 0xFF) return unsupported(o, i >= len ? "truncated header" : "data between markers");
    while (i < len && d[i] == 0xFF) ++i;
    if (i >= len) return unsupported(o, "truncated header");
    const int m = d[i++];
    if (m == 0xD9) return unsupported(o, "EOI before any scan");
    if (m == 0x00 || m == 0x01 || m == 0xD8 || (m >= 0xD0 && m <= 0xD7))
      return unsupported(o, "unexpected marker 0x%02X in the header", m);
    if (i + 2 > len) return unsupported(o, "truncated header");
    const int seglen = d[i] << 8 | d[i + 1];
    if (seglen < 2 || i + seglen > len) return unsupported(o, "a segment runs past the end of the file");
    const uint8_t* s = d + i + 2;
    const int sl = seglen - 2;
    i += seglen;
    if (m == 0xC0 || m == 0xC1) {
      if (have_sof) return unsupported(o, "more than one frame header");
      if (sl < 6) return unsupported(o, "short frame header");
      if (s[0] != 8) return unsupported(o, "%d-bit samples (only 8-bit is decoded on the device)", s[0]);
      H = s[1] << 8 | s[2];
      W = s[3] << 8 | s[4];
      nf = s[5];
      if (sl != 6 + 3 * nf) return unsupported(o, "frame header length does not match its component count");
      if (nf == 4) return unsupported(o, "4 components (CMYK / YCCK)");
      if (nf != 1 && nf != 3) return unsupported(o, "%d components", nf);
      if (H == 0) return unsupported(o, "height given by a DNL marker");
      if (W == 0) return unsupported(o, "zero width");
      if ((int64_t)W * H > kMaxPixels) return unsupported(o, "image larger than 2^28 pixels");
      for (int c = 0; c < nf; ++c) {
        ids[c] = s[6 + 3 * c];
        hs[c] = s[7 + 3 * c] >> 4;
        vs[c] = s[7 + 3 * c] & 15;
        tq[c] = s[8 + 3 * c];
        if (hs[c] < 1 || hs[c] > 4 || vs[c] < 1 || vs[c] > 4) return unsupported(o, "invalid sampling factors");
        if (tq[c] > 3) return unsupported(o, "invalid quantisation table index");
        for (int e = 0; e < c; ++e)
          if (ids[e] == ids[c]) return unsupported(o, "duplicate component id");
      }
      have_sof = true;
    } else if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) {
      return unsupported(o, "progressive JPEG");
    } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) {
      return unsupported(o, "lossless JPEG");
    } else if (m == 0xC5) {
      return unsupported(o, "hierarchical JPEG");
    } else if (m == 0xC9 || m == 0xCC || m == 0xCD) {
      return unsupported(o, "arithmetic coding");
    } else if (m == 0xC8 || (m >= 0xF0 && m <= 0xFD) || (m >= 0x02 && m <= 0xBF)) {
      return unsupported(o, "unsupported marker 0x%02X", m);
    } else if (m == 0xC4) {
      int k = 0;
      while (k < sl) {
        if (k + 17 > sl) return unsupported(o, "truncated Huffman table");
        const int tc = s[k] >> 4, th = s[k] & 15;
        if (tc > 1 || th > 3) return unsupported(o, "invalid Huffman table class or index");
        HuffTable& t = ht[tc][th];
        int total = 0;
        for (int l = 0; l < 16; ++l) total += t.bits[l] = s[k + 1 + l];
        if (total > 256 || k + 17 + total > sl) return unsupported(o, "Huffman table longer than its segment");
        memcpy(t.vals, s + k + 17, total);
        t.nvals = total;
        // libjpeg's code-space check, plus: no all-1s code (the device decoder takes < 8 trailing 1s of a restart
        // interval as padding, which requires that no code looks like it)
        int64_t code = 0;
        for (int l = 1; l <= 16; ++l) {
          code += t.bits[l - 1];
          if (code > ((int64_t)1 << l)) return unsupported(o, "Huffman table overflows its code space");
          if (t.bits[l - 1] && code == ((int64_t)1 << l)) return unsupported(o, "Huffman table with an all-1s code");
          code <<= 1;
        }
        if (tc == 0) {
          if (total > 16) return unsupported(o, "DC Huffman table with more than 16 symbols");
          for (int v = 0; v < total; ++v)
            if (t.vals[v] > 11) return unsupported(o, "DC category above 11 in an 8-bit file");
        }
        t.set = true;
        k += 17 + total;
      }
    } else if (m == 0xDB) {
      int k = 0;
      while (k < sl) {
        const int pq = s[k] >> 4, t = s[k] & 15;
        if (pq > 1 || t > 3) return unsupported(o, "invalid quantisation table");
        if (k + 1 + 64 * (pq + 1) > sl) return unsupported(o, "truncated quantisation table");
        for (int e = 0; e < 64; ++e)
          qt[t][kZigzagHost[e]] = pq ? (uint16_t)(s[k + 1 + 2 * e] << 8 | s[k + 2 + 2 * e]) : s[k + 1 + e];
        qset[t] = true;
        k += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {
      if (sl != 2) return unsupported(o, "invalid DRI segment");
      o->restart_interval = s[0] << 8 | s[1];
    } else if (m == 0xDC) {
      return unsupported(o, "DNL marker");
    } else if (m == 0xE0) {
      if (sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;   // libjpeg's examine_app0
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) {               // libjpeg's examine_app14
        adobe = true;
        adobe_transform = s[11];
      }
    } else if (m == 0xDA) {
      if (!have_sof) return unsupported(o, "scan before the frame header");
      if (sl < 1) return unsupported(o, "short scan header");
      const int ns = s[0];
      if (sl != 1 + 2 * ns + 3) return unsupported(o, "scan header length does not match its component count");
      if (ns != nf) return unsupported(o, "multi-scan file (the first scan does not hold every component)");
      for (int c = 0; c < ns; ++c) {
        if (s[1 + 2 * c] != ids[c]) return unsupported(o, "scan components not in frame order");
        const int td = s[2 + 2 * c] >> 4, ta = s[2 + 2 * c] & 15;
        if (td > 3 || ta > 3 || !ht[0][td].set || !ht[1][ta].set)
          return unsupported(o, "scan uses an undefined Huffman table");
        memcpy(o->dc_bits[c], ht[0][td].bits, 16);
        memcpy(o->dc_vals[c], ht[0][td].vals, 16);
        memcpy(o->ac_bits[c], ht[1][ta].bits, 16);
        memcpy(o->ac_vals[c], ht[1][ta].vals, 256);
        if (!qset[tq[c]]) return unsupported(o, "undefined quantisation table");
        memcpy(o->quant[c], qt[tq[c]], sizeof(o->quant[c]));
      }
      const uint8_t* tail = s + 1 + 2 * ns;
      if (tail[0] != 0 || tail[1] != 63 || tail[2] != 0) return unsupported(o, "scan is not a sequential 0..63 scan");
      break;
    }
    // APPn, COM: skipped
  }
  // the entropy-coded segment ends at the first marker other than RSTn (fill 0xFFs before it belong to the marker)
  const int64_t begin = i;
  int64_t end = -1;
  int code = -1;
  for (int64_t j = i; j < len;) {
    const void* f = memchr(d + j, 0xFF, (size_t)(len - j));
    if (!f) break;
    j = (const uint8_t*)f - d;
    int64_t k = j + 1;
    while (k < len && d[k] == 0xFF) ++k;
    if (k >= len) break;
    if (d[k] == 0x00 || (d[k] >= 0xD0 && d[k] <= 0xD7)) {
      j = k + 1;
      continue;
    }
    end = j;
    code = d[k];
    break;
  }
  if (end < 0) return unsupported(o, "no EOI marker (truncated file)");
  if (code == 0xDC) return unsupported(o, "DNL marker");
  if (code != 0xD9) return unsupported(o, "multi-scan file or marker 0x%02X after the scan", code);
  if (end - begin > kMaxScanBytes) return unsupported(o, "entropy-coded segment larger than 128 MiB");

  int hmax = 1, vmax = 1;
  for (int c = 0; c < nf; ++c) {
    hmax = std::max(hmax, hs[c]);
    vmax = std::max(vmax, vs[c]);
  }
  int bpm = 0;
  if (nf == 3) {
    for (int c = 0; c < 3; ++c) {
      if (hmax % hs[c] || vmax % vs[c]) return unsupported(o, "non-integral sampling ratio");
      const int hr = hmax / hs[c], vr = vmax / vs[c];
      if (!((hr == 1 && vr == 1) || (hr == 2 && vr == 1) || (hr == 2 && vr == 2)))
        return unsupported(o, "sampling ratio other than 1x1, 2x1 or 2x2 (4:4:0, 4:1:1, ...)");
      bpm += hs[c] * vs[c];
    }
    if (bpm > 10) return unsupported(o, "more than 10 blocks per MCU");
    if (jfif) {
    } else if (adobe) {
      if (adobe_transform == 0) return unsupported(o, "RGB colour space (Adobe transform 0)");
      if (adobe_transform != 1) return unsupported(o, "Adobe transform %d", adobe_transform);
    } else if (ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B') {
      return unsupported(o, "RGB colour space (component ids R, G, B)");
    }
    o->mcus_x = (W + 8 * hmax - 1) / (8 * hmax);
    o->mcus_y = (H + 8 * vmax - 1) / (8 * vmax);
  } else {
    bpm = 1;
    o->mcus_x = (W + 7) / 8;
    o->mcus_y = (H + 7) / 8;
  }
  o->supported = 1;
  snprintf(o->reason, sizeof(o->reason), "supported");
  o->width = W;
  o->height = H;
  o->ncomp = nf;
  for (int c = 0; c < nf; ++c) {
    o->h_samp[c] = hs[c];
    o->v_samp[c] = vs[c];
  }
  o->blocks_per_mcu = bpm;
  o->scan_begin = begin;
  o->scan_end = end;
  return YB_OK;
}

extern "C" size_t yb_jpeg_workspace_bytes(int n, const yb_jpeg_info* infos) {
  if (n <= 0 || !infos) return 0;
  return (size_t)batch_size(n, infos).bytes;
}

extern "C" int yb_jpeg_decode(int n, const yb_jpeg_info* infos, const void* src_dev, uint8_t* const* dst_dev,
                              int32_t* status_dev, void* workspace_dev, size_t workspace_bytes, void* stream) {
  YB_REQUIRE(n > 0 && infos && src_dev && dst_dev && status_dev && workspace_dev, "yb_jpeg_decode: null/empty arguments");
  YB_REQUIRE(((uintptr_t)src_dev & 15) == 0 && ((uintptr_t)workspace_dev & 255) == 0,
             "yb_jpeg_decode: src must be 16-byte and the workspace 256-byte aligned");
  for (int i = 0; i < n; ++i) {
    YB_REQUIRE(infos[i].supported == 1, "yb_jpeg_decode: image %d is not supported: %.92s", i, infos[i].reason);
    YB_REQUIRE(infos[i].data_offset >= (int64_t)n * (int64_t)sizeof(yb_jpeg_info) && dst_dev[i],
               "yb_jpeg_decode: image %d: data_offset overlaps the info array, or no destination", i);
  }
  const BatchSize s = batch_size(n, infos);
  YB_REQUIRE(workspace_bytes >= (size_t)s.bytes, "yb_jpeg_decode: workspace %zu < %lld bytes", workspace_bytes,
             (long long)s.bytes);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint8_t* src = static_cast<const uint8_t*>(src_dev);
  uint8_t* ws = static_cast<uint8_t*>(workspace_dev);
  YB_CHECK_CUDA(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * n, st));
  YB_CHECK_CUDA(cudaMemsetAsync(ws, 0, (size_t)s.bytes, st));
  jpeg_setup_kernel<<<1, 1024, 0, st>>>(n, src, ws);
  jpeg_destuff_count_kernel<<<s.tiles, kTileThreads, 0, st>>>(n, src, ws);
  jpeg_destuff_scan_kernel<<<n, 32, 0, st>>>(n, ws, status_dev);
  jpeg_destuff_write_kernel<<<s.tiles, kTileThreads, 0, st>>>(n, src, ws, status_dev);
  YB_CHECK_CUDA(cudaGetLastError());

  int per_sm = 0;
  YB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jpeg_huffman_kernel, kSubThreads, 0));
  YB_REQUIRE(per_sm > 0, "yb_jpeg_decode: the Huffman kernel cannot be resident");
  int grid = std::min<int64_t>(s.items, (int64_t)per_sm * yb::num_sms());
  int total_items = s.items, max_rounds = s.max_nsub + 1;
  const uint8_t* src_arg = src;
  void* args[] = {&n, &total_items, &max_rounds, &src_arg, &ws, &status_dev};
  YB_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)jpeg_huffman_kernel, grid, kSubThreads, args, 0, st));

  jpeg_idct_kernel<<<cdiv(s.blocks, 128), 128, 0, st>>>(n, s.blocks, src, ws, status_dev);
  YB_CHECK_CUDA(cudaGetLastError());

  int64_t px = 0;
  for (int first = 0; first < n; first += kMaxDstPerLaunch) {
    const int count = std::min(kMaxDstPerLaunch, n - first);
    DstPtrs p;
    int64_t chunk = 0;
    for (int k = 0; k < count; ++k) {
      p.dst[k] = dst_dev[first + k];
      chunk += (int64_t)infos[first + k].width * infos[first + k].height;
    }
    const int64_t blocks = std::min<int64_t>((chunk + 255) / 256, (int64_t)yb::num_sms() * 16);
    jpeg_color_kernel<<<(int)std::max<int64_t>(blocks, 1), 256, 0, st>>>(n, first, count, px, px + chunk, ws, p);
    px += chunk;
  }
  YB_CHECK_CUDA(cudaGetLastError());
  return YB_OK;
}
