// Image-space masks of the save-results loop (the reference's gdrn_save_result_of_dataset): paste each ROI's 64x64 mask
// probabilities into the image as detectron2's GPU paste_masks_in_image does, threshold, and encode the result as a
// COCO compressed RLE string (pycocotools rleEncode + rleToString), all on the device; plus the decode + confusion
// counts of the reference's mask tools (compute_mIoU_mask.py, compute_f1_score_mask.py).
//
// Paste arithmetic (detectron2 _do_paste_mask with skip_empty=False, then F.grid_sample(bilinear, zeros,
// align_corners=False)), every step one float32 IEEE operation:
//   gx = ((x + 0.5) - x0) / (x1 - x0) * 2 - 1                   (one torch op per step, never contracted)
//   ix = ((gx + 1) * mw - 1) / 2                                  (grid_sampler_unnormalize)
//   taps floor(ix), floor(ix) + 1; weights (ix_se - ix) * (iy_se - iy), ...; accumulated nw, ne, sw, se with zero
//   padding; pixel = (value >= threshold).
// torch's sm_90 build of grid_sampler_2d_kernel<float> contracts both `(g + 1) * size - 1` (FFMA(size, g + 1, -1), then
// * 0.5) and the four-tap accumulation (an FFMA chain from 0) into FMAs; kUnnormFma / kAccumFma restate that, and
// tests/test_save_results.py holds the paste bit-identical to torch's grid_sample on the H100.
//
// With threshold > 0 only pixels whose taps reach the map can be non-zero: ix in (-1, mw) means the pixel centre lies
// within half a texel of the box.  The kernels evaluate the column / row range of the box widened by one texel and two
// pixels (in float64, clamped to the image) and treat every other pixel as 0.
//
// RLE: run boundaries in Fortran order (pixel index x * H + y), one warp per column, 32 rows per ballot.  A boundary is
// an index k with m[k] != m[k - 1] (m[-1] = 0); boundary words go to a bit workspace (bit y of column x = index
// x * H + y, y in [0, H]: bit H is the step into column x + 1).  Counts are the differences of 0, the boundaries and
// H * W, so the first count is 0 when pixel (0, 0) is set.  Each count x is written as rleToString does: for i > 2
// subtract cnts[i - 2], then 5-bit groups from the low end, 0x20 = more follows, a final group with 0x10 set means a
// negative remainder, each char + 48.
//
// Bound of one string: chars(d) <= 1 + max(c_i, c_{i-2}) / 16 for the delta d of count c_i (one char holds -16..15, every
// further char multiplies the range by 32), so a string of K + 1 counts summing to H * W takes at most
// (K + 1) + 2 * H * W / 16 chars, and K <= H * W.  gdrn_mask_rle_max_chars(H, W) = H * W + H * W / 8 + 2.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxMapElems = 12288;   // 48 KB of shared memory
constexpr int kPasteTile = 4096;      // pixels per block of the bool paste
constexpr int kTileWords = kThreads;  // boundary words per tile of the encoder
constexpr bool kUnnormFma = true;
constexpr bool kAccumFma = true;

struct Box { float x0, y0, x1, y1; };
struct Rect { int c0, c1, r0, r1; };

__device__ __forceinline__ Box box_xyxy(const float* __restrict__ b, int i) {
  return {b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]};
}

// inst_rois = roi_center -/+ scale / 2 in float32
__device__ __forceinline__ Box box_center_scale(const float* __restrict__ c, const float* __restrict__ s, int i) {
  const float h = __fdiv_rn(s[i], 2.f);
  return {__fsub_rn(c[2 * i], h), __fsub_rn(c[2 * i + 1], h), __fadd_rn(c[2 * i], h), __fadd_rn(c[2 * i + 1], h)};
}

__device__ __forceinline__ void axis_range(float a, float b, int m, int size, int& lo_out, int& hi_out) {
  const double lo = fmin((double)a, (double)b), hi = fmax((double)a, (double)b), tex = (hi - lo) / m;
  const double l = fmin(fmax(floor(lo - tex - 2.0), 0.0), (double)size);   // fmin / fmax drop NaN: full range
  const double h = fmin(fmax(ceil(hi + tex + 2.0), 0.0), (double)size);
  lo_out = (int)l;
  hi_out = (int)h > (int)l ? (int)h : (int)l;
}

__device__ __forceinline__ Rect active_rect(const Box& b, int mh, int mw, int H, int W) {
  Rect r;
  axis_range(b.x0, b.x1, mw, W, r.c0, r.c1);
  axis_range(b.y0, b.y1, mh, H, r.r0, r.r1);
  return r;
}

// detectron2's grid value of pixel centre p on one axis
__device__ __forceinline__ float grid_coord(int p, float a0, float a1) {
  return __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn((float)p + 0.5f, a0), __fsub_rn(a1, a0)), 2.f), 1.f);
}

__device__ __forceinline__ float unnormalize(float g, int size) {
  const float t = kUnnormFma ? __fmaf_rn(__fadd_rn(g, 1.f), (float)size, -1.f)
                             : __fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), (float)size), 1.f);
  return __fdiv_rn(t, 2.f);
}

__device__ __forceinline__ float accum(float acc, float v, float w) {
  return kAccumFma ? __fmaf_rn(v, w, acc) : __fadd_rn(acc, __fmul_rn(v, w));
}

// grid_sample of map [mh, mw] (shared memory) at pixel (x, y) of the image
__device__ __forceinline__ float sample(const float* __restrict__ map, int mh, int mw, const Box& b, int x, int y) {
  const float ix = unnormalize(grid_coord(x, b.x0, b.x1), mw);
  const float iy = unnormalize(grid_coord(y, b.y0, b.y1), mh);
  const int ix_nw = (int)floorf(ix), iy_nw = (int)floorf(iy);
  const int ix_se = ix_nw + 1, iy_se = iy_nw + 1;
  const float nw = __fmul_rn(__fsub_rn((float)ix_se, ix), __fsub_rn((float)iy_se, iy));
  const float ne = __fmul_rn(__fsub_rn(ix, (float)ix_nw), __fsub_rn((float)iy_se, iy));
  const float sw = __fmul_rn(__fsub_rn((float)ix_se, ix), __fsub_rn(iy, (float)iy_nw));
  const float se = __fmul_rn(__fsub_rn(ix, (float)ix_nw), __fsub_rn(iy, (float)iy_nw));
  const bool x0in = ix_nw >= 0 && ix_nw < mw, x1in = ix_se >= 0 && ix_se < mw;
  const bool y0in = iy_nw >= 0 && iy_nw < mh, y1in = iy_se >= 0 && iy_se < mh;
  float acc = 0.f;
  if (y0in && x0in) acc = accum(acc, map[iy_nw * mw + ix_nw], nw);
  if (y0in && x1in) acc = accum(acc, map[iy_nw * mw + ix_se], ne);
  if (y1in && x0in) acc = accum(acc, map[iy_se * mw + ix_nw], sw);
  if (y1in && x1in) acc = accum(acc, map[iy_se * mw + ix_se], se);
  return acc;
}

// torch.max / torch.min propagate NaN
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || a < b) ? a : b; }

// The map of one ROI as probabilities in shared memory: mode 0 as given, 1 = L1 ((p - min) / (max - min) over the
// map), 2 = sigmoid (1 / (1 + exp(-p)), torch's CUDA sigmoid).  Every thread of the block calls it.
__device__ void load_prob_map(const float* __restrict__ raw, int m, int mode, float* s_map) {
  __shared__ float s_mn[kWarps], s_mx[kWarps];
  float mn = INFINITY, mx = -INFINITY;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const float v = raw[i];
    s_map[i] = v;
    mn = nan_min(v, mn);
    mx = nan_max(v, mx);
  }
  if (mode == 1) {
    for (int o = 16; o > 0; o >>= 1) {
      mn = nan_min(__shfl_xor_sync(0xffffffffu, mn, o), mn);
      mx = nan_max(__shfl_xor_sync(0xffffffffu, mx, o), mx);
    }
    if ((threadIdx.x & 31) == 0) { s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
  }
  __syncthreads();
  if (mode == 1) {
    mn = s_mn[0];
    mx = s_mx[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { mn = nan_min(s_mn[w], mn); mx = nan_max(s_mx[w], mx); }
  }
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const float v = s_map[i];
    if (mode == 1) s_map[i] = __fdiv_rn(__fsub_rn(v, mn), __fsub_rn(mx, mn));
    else if (mode == 2) s_map[i] = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v)));
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------- bool paste
__global__ void __launch_bounds__(kThreads)
mask_paste_kernel(const float* __restrict__ maps, int mh, int mw, int mode, const float* __restrict__ boxes, int H,
                  int W, float thr, uint8_t* __restrict__ out) {
  extern __shared__ float s_map[];
  const int i = blockIdx.x;
  const long long HW = (long long)H * W;
  const long long p0 = (long long)blockIdx.y * kPasteTile;
  const long long p1 = p0 + kPasteTile < HW ? p0 + kPasteTile : HW;
  uint8_t* o = out + (size_t)i * HW;
  const Box b = box_xyxy(boxes, i);
  const Rect r = active_rect(b, mh, mw, H, W);
  const int ty0 = (int)(p0 / W), ty1 = (int)((p1 - 1) / W);
  if (r.c0 >= r.c1 || r.r0 >= r.r1 || ty1 < r.r0 || ty0 >= r.r1) {   // block-uniform
    for (long long p = p0 + threadIdx.x; p < p1; p += blockDim.x) o[p] = 0;
    return;
  }
  load_prob_map(maps + (size_t)i * mh * mw, mh * mw, mode, s_map);
  for (long long p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    uint8_t v = 0;
    if (x >= r.c0 && x < r.c1 && y >= r.r0 && y < r.r1) v = sample(s_map, mh, mw, b, x, y) >= thr;
    o[p] = v;
  }
}

// ---------------------------------------------------------------------------------------------- run boundaries
// String s = kind * n + roi (kind 0: maps0, kind 1: maps1).  One warp per column of the active range.
__global__ void __launch_bounds__(kThreads)
mask_runs_kernel(const float* __restrict__ maps0, const float* __restrict__ maps1, int n, int mh, int mw, int mode,
                 const float* __restrict__ roi_center, const float* __restrict__ scale, int H, int W, float thr,
                 uint32_t* __restrict__ bits) {
  extern __shared__ float s_map[];
  const int s = blockIdx.x, roi = s % n;
  const Box b = box_center_scale(roi_center, scale, roi);
  const Rect r = active_rect(b, mh, mw, H, W);
  const int ncols = r.c1 - r.c0;
  if (r.r0 >= r.r1 || (int)blockIdx.y * kWarps >= ncols) return;   // block-uniform
  load_prob_map((s < n ? maps0 : maps1) + (size_t)roi * mh * mw, mh * mw, mode, s_map);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwc = (H >> 5) + 1;
  const bool chain = r.r0 == 0 && r.r1 == H;   // the last row of a column and the first of the next are both active
  for (int c = blockIdx.y * kWarps + warp; c < ncols; c += gridDim.y * kWarps) {
    const int x = r.c0 + c;
    // value entering the column's range: the previous column's last row when the columns chain, else 0
    int prev = 0;
    if (chain && c > 0) prev = sample(s_map, mh, mw, b, x - 1, H - 1) >= thr;
    // the step just past the range (index x * H + r1) is this column's unless the next column starts there
    const bool end_here = (r.r1 < H) || (x + 1 < W && (r.r0 > 0 || x + 1 == r.c1));
    uint32_t* col = bits + ((size_t)s * W + x) * nwc;
    for (int j = r.r0 >> 5; j <= (r.r1 >> 5) && j < nwc; ++j) {
      const int y = 32 * j + lane;
      const bool active = y >= r.r0 && y < r.r1;
      const int v = active ? (sample(s_map, mh, mw, b, x, y) >= thr) : 0;
      int pv = __shfl_up_sync(0xffffffffu, v, 1);
      if (lane == 0) pv = prev;
      const bool flag = (active && v != pv) || (y == r.r1 && end_here && pv == 1);
      const uint32_t word = __ballot_sync(0xffffffffu, flag);
      if (lane == 0) col[j] = word;
      prev = __shfl_sync(0xffffffffu, v, 31);
    }
  }
}

// ---------------------------------------------------------------------------------------------- counts -> chars
__device__ __forceinline__ int rle_nchars(long long x) {
  int k = 0;
  bool more = true;
  while (more) {
    const long long c = x & 0x1f;
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    ++k;
  }
  return k;
}

__device__ __forceinline__ int rle_put(long long x, char* __restrict__ o) {
  int k = 0;
  bool more = true;
  while (more) {
    long long c = x & 0x1f;
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    o[k++] = (char)(c + 48);
  }
  return k;
}

// exclusive block scan of one value per thread; *total = the sum (every thread)
template <typename T>
__device__ __forceinline__ T block_excl_scan(T v, T* total) {
  __shared__ T s_w[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) s_w[warp] = inc;
  __syncthreads();
  T before = 0, all = 0;
  for (int w = 0; w < kWarps; ++w) {
    const T t = s_w[w];
    if (w < warp) before += t;
    all += t;
  }
  __syncthreads();
  *total = all;
  return before + inc - v;
}

// One block per string.  WRITE = false: string lengths -> lens[s].  WRITE = true: offsets from lens (strings packed in
// string order), table[s] = (offset, length) and the chars.
template <bool WRITE>
__global__ void __launch_bounds__(kThreads)
mask_rle_kernel(int n, int mh, int mw, const float* __restrict__ roi_center, const float* __restrict__ scale, int H,
                int W, const uint32_t* __restrict__ bits, long long* __restrict__ lens, char* __restrict__ chars,
                long long* __restrict__ table) {
  __shared__ int s_pos[3 + 32 * kTileWords];   // the three boundaries before the tile, then the tile's
  const int s = blockIdx.x, tid = threadIdx.x;
  const Box b = box_center_scale(roi_center, scale, s % n);
  const Rect r = active_rect(b, mh, mw, H, W);
  const int nwc = (H >> 5) + 1;
  const int j0 = r.r0 >> 5, j1 = min(r.r1 >> 5, nwc - 1);
  const int nw = j1 - j0 + 1;
  const long long total_words = (r.r0 < r.r1 && r.c0 < r.c1) ? (long long)(r.c1 - r.c0) * nw : 0;
  const long long HW = (long long)H * W;
  long long base = 0;
  if (WRITE) {
    long long part = 0, sum;
    for (int t = tid; t < s; t += kThreads) part += lens[t];
    block_excl_scan(part, &sum);
    base = sum;
  }
  if (tid < 3) s_pos[tid] = 0;   // B_0 = 0; the two before it are never read (no delta for counts 0..2)
  __syncthreads();
  long long nb = 0, nchars = 0;   // boundaries and chars before the tile
  for (long long t0 = 0; t0 < total_words; t0 += kTileWords) {
    const long long w = t0 + tid;
    uint32_t word = 0;
    int pos0 = 0;
    if (w < total_words) {
      const int x = r.c0 + (int)(w / nw), j = j0 + (int)(w % nw);
      word = bits[((size_t)s * W + x) * nwc + j];
      pos0 = x * H + 32 * j;
    }
    int T;
    const int off = block_excl_scan((int)__popc(word), &T);
    for (int k = 0; word; ++k) {
      const int bit = __ffs(word) - 1;
      word &= word - 1;
      s_pos[3 + off + k] = pos0 + bit;
    }
    __syncthreads();
    const int per = (T + kThreads - 1) / kThreads;
    const int i0 = min(T, tid * per), i1 = min(T, i0 + per);
    long long len = 0;
    for (int i = i0; i < i1; ++i) {
      long long x = s_pos[3 + i] - s_pos[2 + i];
      if (nb + i > 2) x -= s_pos[1 + i] - s_pos[i];
      len += rle_nchars(x);
    }
    long long L;
    const long long lo = block_excl_scan(len, &L);
    if (WRITE) {
      char* o = chars + base + nchars + lo;
      for (int i = i0; i < i1; ++i) {
        long long x = s_pos[3 + i] - s_pos[2 + i];
        if (nb + i > 2) x -= s_pos[1 + i] - s_pos[i];
        o += rle_put(x, o);
      }
    }
    int keep = 0;
    if (tid < 3) keep = s_pos[T + tid];
    __syncthreads();
    if (tid < 3) s_pos[tid] = keep;
    __syncthreads();
    nb += T;
    nchars += L;
  }
  if (tid == 0) {   // the last count: H * W - B_K
    long long x = HW - s_pos[2];
    if (nb > 2) x -= s_pos[1] - s_pos[0];
    const long long total = nchars + (WRITE ? rle_put(x, chars + base + nchars) : rle_nchars(x));
    if (WRITE) {
      table[2 * s] = base;
      table[2 * s + 1] = total;
    } else {
      lens[s] = total;
    }
  }
}

// ---------------------------------------------------------------------------------------------- decode + confusion
// status: 0 ok, 1 a group runs past the end of the string, 2 a char outside '0'..'o', 3 a group of more than 7 chars,
// 4 a negative count or a total past H * W, 5 a total short of H * W, 6 (offset, length) outside the char buffer
constexpr int kRunChunk = 1024;

__global__ void __launch_bounds__(kThreads)
rle_confusion_kernel(const char* __restrict__ chars, long long chars_bytes, const long long* __restrict__ table,
                     const uint8_t* __restrict__ gt, int H, int W, int* __restrict__ status_out,
                     long long* __restrict__ counts) {
  __shared__ int s_run[2 * kRunChunk];
  __shared__ int s_nrun, s_done;
  const int s = blockIdx.x, tid = threadIdx.x;
  const long long HW = (long long)H * W;
  const uint8_t* g = gt + (size_t)s * HW;
  long long g1 = 0;
  for (long long k = tid; k < HW; k += kThreads) g1 += g[k] != 0;
  // parser state (thread 0)
  const long long off = table[2 * s], len = table[2 * s + 1];
  int status = (off < 0 || len < 0 || off > chars_bytes || len > chars_bytes - off) ? 6 : 0;
  const char* str = chars + (status ? 0 : off);
  long long p = 0, m = 0, pos = 0, c1 = 0, c2 = 0, p1 = 0;   // char, count index, pixels so far, cnts[m-1], cnts[m-2]
  long long tp = 0;
  while (true) {
    if (tid == 0) {
      int nr = 0;
      while (!status && nr < kRunChunk && p < len) {
        unsigned long long x = 0;
        int k = 0;
        bool more = true;
        while (more) {
          if (p >= len) { status = 1; break; }
          const int c = (int)(unsigned char)str[p] - 48;
          if (c < 0 || c > 63) { status = 2; break; }
          if (k == 7) { status = 3; break; }
          x |= (unsigned long long)(c & 0x1f) << (5 * k);
          more = c & 0x20;
          ++p;
          ++k;
          if (!more && (c & 0x10)) x |= ~0ull << (5 * k);
        }
        if (status) break;
        long long v = (long long)x;
        if (m > 2) v += c2;
        if (v < 0 || pos + v > HW) { status = 4; break; }
        c2 = c1;
        c1 = v;
        if (m & 1) {
          s_run[2 * nr] = (int)pos;
          s_run[2 * nr + 1] = (int)(pos + v);
          ++nr;
          p1 += v;
        }
        pos += v;
        ++m;
      }
      const bool done = status || p >= len;
      if (done && !status && pos != HW) status = 5;
      s_nrun = nr;
      s_done = done;
    }
    __syncthreads();
    const int nr = s_nrun, done = s_done;
    const int lane = tid & 31, warp = tid >> 5;
    for (int q = warp; q < nr; q += kWarps) {
      const int a = s_run[2 * q], e = s_run[2 * q + 1];
      for (int k = a + lane; k < e; k += 32) {
        const int x = k / H, y = k - x * H;
        tp += g[(size_t)y * W + x] != 0;
      }
    }
    __syncthreads();
    if (done) break;
  }
  long long TP, G1;
  block_excl_scan(tp, &TP);
  block_excl_scan(g1, &G1);
  if (tid == 0) {
    status_out[s] = status;
    const long long FP = p1 - TP, FN = G1 - TP;
    counts[4 * s] = TP;
    counts[4 * s + 1] = FP;
    counts[4 * s + 2] = FN;
    counts[4 * s + 3] = HW - TP - FP - FN;
  }
}

inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }
inline size_t bits_bytes(int S, int H, int W) { return (size_t)S * W * ((H >> 5) + 1) * sizeof(uint32_t); }
constexpr long long kMaxPixels = 65535LL * kPasteTile;   // one grid row of paste tiles

}  // namespace

extern "C" int gdrn_mask_paste(const float* masks, int n, int mh, int mw, int mode, const float* boxes, int H, int W,
                               float threshold, uint8_t* out, void* stream) {
  GDRN_REQUIRE(n >= 0 && mh > 0 && mw > 0 && mh * mw <= kMaxMapElems, "mask_paste: masks must be [n,mh,mw] with mh*mw <= 12288");
  GDRN_REQUIRE(H > 0 && W > 0 && (long long)H * W <= kMaxPixels, "mask_paste: image must have 1..65535*4096 pixels");
  GDRN_REQUIRE(mode >= 0 && mode <= 2, "mask_paste: mode must be 0 (probabilities), 1 (L1) or 2 (sigmoid)");
  GDRN_REQUIRE(threshold > 0.f, "mask_paste: threshold must be > 0 (detectron2 returns uint8 probabilities otherwise)");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(masks && boxes && out, "mask_paste: null argument");
  const long long tiles = ((long long)H * W + kPasteTile - 1) / kPasteTile;
  mask_paste_kernel<<<dim3((unsigned)n, (unsigned)tiles), kThreads, (size_t)mh * mw * sizeof(float), (cudaStream_t)stream>>>(
      masks, mh, mw, mode, boxes, H, W, threshold, out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" size_t gdrn_mask_rle_max_chars(int H, int W) {
  const size_t hw = (size_t)(H > 0 ? H : 0) * (size_t)(W > 0 ? W : 0);
  return hw + hw / 8 + 2;
}

extern "C" size_t gdrn_mask_rle_workspace_bytes(int S, int H, int W) {
  if (S <= 0 || H <= 0 || W <= 0) return 0;
  return align256(bits_bytes(S, H, W)) + align256((size_t)S * sizeof(long long));
}

extern "C" int gdrn_mask_paste_rle(const float* maps0, const float* maps1, int n, int mh, int mw, int mode,
                                   const float* roi_center, const float* scale, int H, int W, float threshold,
                                   void* workspace, size_t workspace_bytes, char* chars, size_t chars_bytes,
                                   long long* table, void* stream) {
  GDRN_REQUIRE(n >= 0 && mh > 0 && mw > 0 && mh * mw <= kMaxMapElems, "mask_paste_rle: maps must be [n,1,mh,mw] with mh*mw <= 12288");
  GDRN_REQUIRE(H > 0 && W > 0 && (long long)H * W <= kMaxPixels, "mask_paste_rle: image must have 1..65535*4096 pixels");
  GDRN_REQUIRE(mode >= 0 && mode <= 2, "mask_paste_rle: mode must be 0 (probabilities), 1 (L1) or 2 (sigmoid)");
  GDRN_REQUIRE(threshold > 0.f, "mask_paste_rle: threshold must be > 0 (detectron2 returns uint8 probabilities otherwise)");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(maps0 && roi_center && scale && workspace && chars && table, "mask_paste_rle: null argument");
  const int S = maps1 ? 2 * n : n;
  GDRN_REQUIRE(n <= (1 << 29), "mask_paste_rle: too many ROIs");
  GDRN_REQUIRE(workspace_bytes >= gdrn_mask_rle_workspace_bytes(S, H, W), "mask_paste_rle: workspace too small");
  GDRN_REQUIRE(chars_bytes / (size_t)S >= gdrn_mask_rle_max_chars(H, W),
               "mask_paste_rle: chars must hold gdrn_mask_rle_max_chars(H, W) per string");
  uint32_t* bits = (uint32_t*)workspace;
  long long* lens = (long long*)((char*)workspace + align256(bits_bytes(S, H, W)));
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned col_blocks = (unsigned)((W + 4 * kWarps - 1) / (4 * kWarps));
  mask_runs_kernel<<<dim3((unsigned)S, col_blocks), kThreads, (size_t)mh * mw * sizeof(float), st>>>(
      maps0, maps1, n, mh, mw, mode, roi_center, scale, H, W, threshold, bits);
  GDRN_CHECK_CUDA(cudaGetLastError());
  mask_rle_kernel<false><<<S, kThreads, 0, st>>>(n, mh, mw, roi_center, scale, H, W, bits, lens, chars, table);
  GDRN_CHECK_CUDA(cudaGetLastError());
  mask_rle_kernel<true><<<S, kThreads, 0, st>>>(n, mh, mw, roi_center, scale, H, W, bits, lens, chars, table);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(3);
  return GDRN_OK;
}

extern "C" int gdrn_rle_confusion(const char* chars, size_t chars_bytes, const long long* table, int P, const uint8_t* gt,
                                  int H, int W, int* status, long long* counts, void* stream) {
  GDRN_REQUIRE(P >= 0 && H > 0 && W > 0 && (long long)H * W <= kMaxPixels, "rle_confusion: bad shape");
  if (P == 0) return GDRN_OK;
  GDRN_REQUIRE(chars && table && gt && status && counts, "rle_confusion: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  rle_confusion_kernel<<<P, kThreads, 0, st>>>(chars, (long long)chars_bytes, table, gt, H, W, status, counts);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  int* h = (int*)malloc((size_t)P * sizeof(int));
  GDRN_REQUIRE(h != nullptr, "rle_confusion: out of host memory");
  cudaError_t e = cudaMemcpyAsync(h, status, (size_t)P * sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    free(h);
    GDRN_CHECK_CUDA(e);
  }
  static const char* why[] = {"", "a group runs past the end of the string", "a char outside '0'..'o'",
                              "a group of more than 7 chars", "a negative count or more than H*W pixels",
                              "fewer than H*W pixels", "(offset, length) outside the char buffer"};
  for (int i = 0; i < P; ++i) {
    if (h[i] != 0) {
      char msg[160];
      snprintf(msg, sizeof(msg), "rle_confusion: string %d is malformed: %s", i, why[h[i] >= 1 && h[i] <= 6 ? h[i] : 0]);
      free(h);
      gdrn_set_last_error(__FILE__, __LINE__, msg);
      return GDRN_ERR_INVALID;
    }
  }
  free(h);
  return GDRN_OK;
}
