// YOLOX training loss on the GPU: batched SimOTA assignment and the IoU, objectness, class and L1 terms with their
// gradients, for a whole batch in five launches with no host synchronisation between them.
//
// Replaces YOLOXHead.get_losses (det/yolox/models/yolo_head.py:256-426), get_assignments / get_in_boxes_info /
// dynamic_k_matching (:436-627) and IOUloss (det/yolox/models/losses.py).  DESIGN.md §7q pins every rule.
//   1. yl_candidate_kernel   (image, anchor): candidate flag (in any GT's box or 2.5-stride centre region) and the
//      anchor's class-cost sum over all classes against a zero target; GT count and class check per image.
//   2. yl_select_kernel      (image, GT), one CTA: IoU and cost against every candidate, per-thread top-10 lists merged
//      across the CTA, k = max(1, int(sum of the top-10 IoUs)), the k cheapest (cost, anchor) pairs recorded with an
//      atomic match count per anchor.
//   3. yl_resolve_kernel     (image, anchor): anchors matched more than once go to the argmin of their cost over all GTs
//      (recomputed with the same fp32 expression); fg flag, matched GT, IoU target; per-anchor loss terms summed into
//      one fixed-order partial per CTA.
//   4. yl_finalize_kernel    one CTA: the partials in a fixed order -> the four losses, num_fg, the error flag.
//   5. yl_backward_kernel    one thread per gradient element, from the saved assignment and the upstream gradients.
// The candidate test and the pair cost use explicit round-to-nearest intrinsics, so no FMA contraction can make them
// differ from an fp32 replica or between stages 2 and 3.
#include "common.cuh"

namespace {

constexpr int YL_THREADS = 256;
constexpr int YL_TOPK = 10;
constexpr int YL_MAX_GT = 1024;
constexpr int YL_NOFF = 16;

struct YlLayout {
  size_t off[YL_NOFF + 1];
};

inline size_t yl_align(size_t x) { return (x + 255) & ~(size_t)255; }

inline int yl_blocks(int A) { return (A + YL_THREADS - 1) / YL_THREADS; }

YlLayout yl_layout(int B, int A, int M) {
  const size_t BA = (size_t)B * A, BM = (size_t)B * (M > 0 ? M : 1), P = (size_t)B * yl_blocks(A);
  const size_t sz[YL_NOFF] = {
      (size_t)B * 4,         // 0 nlabel [B] i32
      BA,                    // 1 cand [B,A] u8
      BA * 4,                // 2 cls_sum [B,A] f32
      BA * 4,                // 3 count [B,A] i32
      BA * 4,                // 4 chooser [B,A] i32 (lowest GT that chose the anchor)
      (size_t)B * 4,         // 5 n_cand [B] i32
      BM * 4,                // 6 k [B,M] i32
      BM * 4,                // 7 iou_sum [B,M] f32
      BM * YL_TOPK * 4,      // 8 chosen [B,M,10] i32 (-1 padded)
      BA,                    // 9 fg [B,A] u8
      BA * 4,                // 10 matched [B,A] i32 (-1 off fg)
      BA * 4,                // 11 iou_t [B,A] f32
      P * 4 * 4,             // 12 partial [P,4] f32 (iou, obj, cls, l1 sums)
      P * 4,                 // 13 partial_fg [P] i32
      (size_t)B * 4,         // 14 err [B] i32
      8 * 4,                 // 15 result [8] f32
  };
  YlLayout l;
  size_t o = 0;
  for (int i = 0; i < YL_NOFF; ++i) {
    l.off[i] = o;
    o = yl_align(o + sz[i]);
  }
  l.off[YL_NOFF] = o;
  return l;
}

struct YlWs {
  int* nlabel;
  uint8_t* cand;
  float* cls_sum;
  int* count;
  int* chooser;
  int* n_cand;
  int* k;
  float* iou_sum;
  int* chosen;
  uint8_t* fg;
  int* matched;
  float* iou_t;
  float* partial;
  int* partial_fg;
  int* err;
  float* result;
};

YlWs yl_ws(void* workspace, int B, int A, int M) {
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  const YlLayout l = yl_layout(B, A, M);
  YlWs w;
  w.nlabel = reinterpret_cast<int*>(base + l.off[0]);
  w.cand = base + l.off[1];
  w.cls_sum = reinterpret_cast<float*>(base + l.off[2]);
  w.count = reinterpret_cast<int*>(base + l.off[3]);
  w.chooser = reinterpret_cast<int*>(base + l.off[4]);
  w.n_cand = reinterpret_cast<int*>(base + l.off[5]);
  w.k = reinterpret_cast<int*>(base + l.off[6]);
  w.iou_sum = reinterpret_cast<float*>(base + l.off[7]);
  w.chosen = reinterpret_cast<int*>(base + l.off[8]);
  w.fg = base + l.off[9];
  w.matched = reinterpret_cast<int*>(base + l.off[10]);
  w.iou_t = reinterpret_cast<float*>(base + l.off[11]);
  w.partial = reinterpret_cast<float*>(base + l.off[12]);
  w.partial_fg = reinterpret_cast<int*>(base + l.off[13]);
  w.err = reinterpret_cast<int*>(base + l.off[14]);
  w.result = reinterpret_cast<float*>(base + l.off[15]);
  return w;
}

__device__ __forceinline__ float yl_f(float x) { return x; }
__device__ __forceinline__ float yl_f(__half x) { return __half2float(x); }
__device__ __forceinline__ float yl_f(__nv_bfloat16 x) { return __bfloat162float(x); }
template <typename T> __device__ __forceinline__ T yl_to(float x);
template <> __device__ __forceinline__ float yl_to<float>(float x) { return x; }
template <> __device__ __forceinline__ __half yl_to<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 yl_to<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

struct YlGt {
  float cx, cy, w, h;
  int cls;
};

// The image's labels -> shared GT table (first n rows, n = rows with a positive sum); returns n.  Flags a class id
// that F.one_hot would reject (truncated to an integer outside [0, C), or NaN) in *err_out when err_out is non-null.
__device__ int yl_load_gts(const float* __restrict__ labels, int b, int M, int C, YlGt* s_gt, int* s_n, int* err_out) {
  const float* L = labels + (size_t)b * M * 5;
  __shared__ int s_cnt, s_bad;
  if (threadIdx.x == 0) { s_cnt = 0; s_bad = 0; }
  __syncthreads();
  int cnt = 0;
  for (int r = threadIdx.x; r < M; r += blockDim.x) {
    const float* row = L + (size_t)r * 5;
    const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(row[0], row[1]), row[2]), row[3]), row[4]);
    cnt += s > 0.f;
  }
  atomicAdd(&s_cnt, cnt);
  __syncthreads();
  const int n = s_cnt;
  for (int r = threadIdx.x; r < n; r += blockDim.x) {
    const float* row = L + (size_t)r * 5;
    const float c = truncf(row[0]);
    const bool ok = c >= 0.f && c < (float)C;   // false for NaN
    if (!ok) s_bad = 1;
    s_gt[r] = YlGt{row[1], row[2], row[3], row[4], ok ? (int)c : 0};
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *s_n = n;
    if (err_out) *err_out = s_bad;
  }
  __syncthreads();
  return n;
}

// ---- the pair expressions (one rounding per operation) ----
__device__ __forceinline__ float yl_sigmoid(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }
// sqrt(sigmoid(cls) * sigmoid(obj)), the reference's joint score
__device__ __forceinline__ float yl_score(float cls_logit, float sig_obj) {
  return __fsqrt_rn(__fmul_rn(yl_sigmoid(cls_logit), sig_obj));
}
// binary_cross_entropy against 0 / against 1, with torch's log >= -100 clamp
__device__ __forceinline__ float yl_bce0(float p) { return -fmaxf(logf(__fsub_rn(1.f, p)), -100.f); }
__device__ __forceinline__ float yl_bce1(float p) { return -fmaxf(logf(p), -100.f); }

// bboxes_iou(xyxy=False): area_i / (area_a + area_b - area_i), no epsilon.  Evaluated in fp64 and rounded once: in
// fp32 the box edges (c -+ w/2 near 800 px) cancel in br - tl and leave the IoU of small overlaps off by ~1e-6.
__device__ __forceinline__ float yl_iou(const YlGt& g, float px, float py, float pw, float ph) {
  const double gw2 = 0.5 * g.w, gh2 = 0.5 * g.h, pw2 = 0.5 * (double)pw, ph2 = 0.5 * (double)ph;
  const double tlx = fmax(g.cx - gw2, px - pw2), tly = fmax(g.cy - gh2, py - ph2);
  const double brx = fmin(g.cx + gw2, px + pw2), bry = fmin(g.cy + gh2, py + ph2);
  const double inter = (tlx < brx && tly < bry) ? (brx - tlx) * (bry - tly) : 0.0;
  return (float)(inter / ((double)g.w * g.h + (double)pw * ph - inter));
}

// (cls_cost + 3 * -log(iou + 1e-8)): the unpenalised pair cost.  cls_cost = the anchor's sum against a zero target with
// the GT class's term swapped for its term against one.
__device__ __forceinline__ float yl_cost0(float cls_sum, float cls_logit, float sig_obj, float iou) {
  const float p = yl_score(cls_logit, sig_obj);
  const float cls_cost = __fadd_rn(__fsub_rn(cls_sum, yl_bce0(p)), yl_bce1(p));
  return __fadd_rn(cls_cost, __fmul_rn(3.f, -logf(__fadd_rn(iou, 1e-8f))));
}

struct YlAnchor {
  float xc, yc, r;
};
__device__ __forceinline__ YlAnchor yl_anchor(const float* __restrict__ shifts, int A, int a) {
  const float xs = shifts[a], ys = shifts[A + a], st = shifts[2 * A + a];
  const float h = __fmul_rn(0.5f, st);
  return YlAnchor{__fadd_rn(__fmul_rn(xs, st), h), __fadd_rn(__fmul_rn(ys, st), h), __fmul_rn(2.5f, st)};
}
// in the GT's box / in its centre region: all four deltas strictly > 0
__device__ __forceinline__ bool yl_in_box(const YlGt& g, const YlAnchor& an) {
  const float w2 = __fmul_rn(0.5f, g.w), h2 = __fmul_rn(0.5f, g.h);
  return __fsub_rn(an.xc, __fsub_rn(g.cx, w2)) > 0.f && __fsub_rn(an.yc, __fsub_rn(g.cy, h2)) > 0.f &&
         __fsub_rn(__fadd_rn(g.cx, w2), an.xc) > 0.f && __fsub_rn(__fadd_rn(g.cy, h2), an.yc) > 0.f;
}
__device__ __forceinline__ bool yl_in_ctr(const YlGt& g, const YlAnchor& an) {
  return __fsub_rn(an.xc, __fsub_rn(g.cx, an.r)) > 0.f && __fsub_rn(an.yc, __fsub_rn(g.cy, an.r)) > 0.f &&
         __fsub_rn(__fadd_rn(g.cx, an.r), an.xc) > 0.f && __fsub_rn(__fadd_rn(g.cy, an.r), an.yc) > 0.f;
}

template <typename T>
__device__ __forceinline__ float yl_pair_cost(const YlGt& g, const YlAnchor& an, const T* __restrict__ row, float cls_sum,
                                              float sig_obj, float* iou_out, float* cost0_out) {
  const float iou = yl_iou(g, yl_f(row[0]), yl_f(row[1]), yl_f(row[2]), yl_f(row[3]));
  const float c0 = yl_cost0(cls_sum, yl_f(row[5 + g.cls]), sig_obj, iou);
  *iou_out = iou;
  *cost0_out = c0;
  return (yl_in_box(g, an) && yl_in_ctr(g, an)) ? c0 : __fadd_rn(c0, 100000.f);
}

// ---------------------------------------------------------------------------------------------------------- stage 1
template <typename T>
__global__ void __launch_bounds__(YL_THREADS)
yl_candidate_kernel(const T* __restrict__ outputs, const float* __restrict__ labels, const float* __restrict__ shifts, int A,
                    int C, int M, YlWs w) {
  __shared__ YlGt s_gt[YL_MAX_GT];
  __shared__ int s_n;
  const int b = blockIdx.y;
  const int n = yl_load_gts(labels, b, M, C, s_gt, &s_n, blockIdx.x == 0 ? &w.err[b] : nullptr);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    w.nlabel[b] = n;
    w.n_cand[b] = 0;
  }
  const int a = blockIdx.x * YL_THREADS + threadIdx.x;
  if (a >= A) return;
  const YlAnchor an = yl_anchor(shifts, A, a);
  bool cand = false;
  for (int g = 0; g < n && !cand; ++g) cand = yl_in_box(s_gt[g], an) || yl_in_ctr(s_gt[g], an);
  const size_t ba = (size_t)b * A + a;
  float s = 0.f;
  if (cand) {
    const T* row = outputs + ba * (5 + C);
    const float so = yl_sigmoid(yl_f(row[4]));
    for (int c = 0; c < C; ++c) s = __fadd_rn(s, yl_bce0(yl_score(yl_f(row[5 + c]), so)));
  }
  w.cand[ba] = cand;
  w.cls_sum[ba] = s;
  w.count[ba] = 0;
  w.chooser[ba] = 0x7fffffff;
}

// ---------------------------------------------------------------------------------------------------------- stage 2
__device__ __forceinline__ bool yl_less(float c, int i, float c2, int i2) { return c < c2 || (c == c2 && i < i2); }

template <typename T>
__global__ void __launch_bounds__(YL_THREADS)
yl_select_kernel(const T* __restrict__ outputs, const float* __restrict__ labels, const float* __restrict__ shifts, int A,
                 int C, int M, float* __restrict__ trace, YlWs w) {
  const int g = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = w.nlabel[b];
  const size_t bg = (size_t)b * M + g;
  if (g >= n) {   // a padding row: no choice
    if (tid < YL_TOPK) w.chosen[bg * YL_TOPK + tid] = -1;
    if (tid == 0) { w.k[bg] = 0; w.iou_sum[bg] = 0.f; }
    return;
  }
  const float* L = labels + ((size_t)b * M + g) * 5;
  const float cl = truncf(L[0]);
  const YlGt gt{L[1], L[2], L[3], L[4], (cl >= 0.f && cl < (float)C) ? (int)cl : 0};
  // per-thread lists: the 10 cheapest (cost, anchor) and the 10 largest IoUs, sorted
  float lc[YL_TOPK], lv[YL_TOPK];
  int li[YL_TOPK];
#pragma unroll
  for (int j = 0; j < YL_TOPK; ++j) { lc[j] = INFINITY; li[j] = 0x7fffffff; lv[j] = -INFINITY; }
  int n_cand = 0;
  for (int a = tid; a < A; a += YL_THREADS) {
    const size_t ba = (size_t)b * A + a;
    if (!w.cand[ba]) continue;
    ++n_cand;
    const T* row = outputs + ba * (5 + C);
    float iou, c0;
    float c = yl_pair_cost(gt, yl_anchor(shifts, A, a), row, w.cls_sum[ba], yl_sigmoid(yl_f(row[4])), &iou, &c0);
    if (trace) {
      float* t = trace + (((size_t)b * M + g) * A + a) * 3;
      t[0] = iou; t[1] = c0; t[2] = c;
    }
    int i = a;
    float v = iou;
#pragma unroll
    for (int j = 0; j < YL_TOPK; ++j) {
      if (yl_less(c, i, lc[j], li[j])) {
        const float tc = lc[j]; const int ti = li[j];
        lc[j] = c; li[j] = i; c = tc; i = ti;
      }
      if (v > lv[j]) { const float tv = lv[j]; lv[j] = v; v = tv; }
    }
  }
  __shared__ float s_c[YL_THREADS / 32], s_v[YL_THREADS / 32];
  __shared__ int s_i[YL_THREADS / 32], s_t[YL_THREADS / 32], s_cnt[YL_THREADS / 32];
  __shared__ int s_sel[YL_TOPK];
  __shared__ float s_top[YL_TOPK];
#pragma unroll
  for (int o = 16; o; o >>= 1) n_cand += __shfl_xor_sync(0xffffffffu, n_cand, o);
  if (lane == 0) s_cnt[warp] = n_cand;
  __syncthreads();
  int total = 0;
  for (int k = 0; k < YL_THREADS / 32; ++k) total += s_cnt[k];
  const int n_top = min(YL_TOPK, total);
  // merge: one CTA-wide (cost, anchor) argmin and one (IoU, thread) argmax per round; the winners pop their heads
  for (int r = 0; r < YL_TOPK; ++r) {
    float c = lc[0], v = lv[0];
    int i = li[0], t = tid;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float c2 = __shfl_xor_sync(0xffffffffu, c, o), v2 = __shfl_xor_sync(0xffffffffu, v, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, i, o), t2 = __shfl_xor_sync(0xffffffffu, t, o);
      if (yl_less(c2, i2, c, i)) { c = c2; i = i2; }
      if (v2 > v || (v2 == v && t2 < t)) { v = v2; t = t2; }
    }
    if (lane == 0) { s_c[warp] = c; s_i[warp] = i; s_v[warp] = v; s_t[warp] = t; }
    __syncthreads();
    c = s_c[0]; i = s_i[0]; v = s_v[0]; t = s_t[0];
    for (int k = 1; k < YL_THREADS / 32; ++k) {
      if (yl_less(s_c[k], s_i[k], c, i)) { c = s_c[k]; i = s_i[k]; }
      if (s_v[k] > v || (s_v[k] == v && s_t[k] < t)) { v = s_v[k]; t = s_t[k]; }
    }
    if (tid == 0) { s_sel[r] = i; s_top[r] = v; }
    const bool pop_c = li[0] == i && i != 0x7fffffff, pop_v = t == tid;
#pragma unroll
    for (int j = 0; j < YL_TOPK - 1; ++j) {
      if (pop_c) { lc[j] = lc[j + 1]; li[j] = li[j + 1]; }
      if (pop_v) lv[j] = lv[j + 1];
    }
    if (pop_c) { lc[YL_TOPK - 1] = INFINITY; li[YL_TOPK - 1] = 0x7fffffff; }
    if (pop_v) lv[YL_TOPK - 1] = -INFINITY;
    __syncthreads();
  }
  if (tid == 0) {
    float s = 0.f;
    for (int r = 0; r < n_top; ++r) s = __fadd_rn(s, s_top[r]);
    // k = max(1, int(sum)); no candidate at all: the GT takes nothing
    const int k = total == 0 ? 0 : min(max(1, (int)s), total);
    w.k[bg] = k;
    w.iou_sum[bg] = s;
    if (g == 0) w.n_cand[b] = total;
    for (int r = 0; r < YL_TOPK; ++r) {
      const int a = r < k ? s_sel[r] : -1;
      w.chosen[bg * YL_TOPK + r] = a;
      if (a >= 0) {
        atomicAdd(&w.count[(size_t)b * A + a], 1);
        atomicMin(&w.chooser[(size_t)b * A + a], g);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- stage 3
__device__ __forceinline__ float yl_bce_logits(float x, float y) {
  // (1 - y) x + log(1 + exp(-x)), in the overflow-safe form
  return __fadd_rn(__fsub_rn(fmaxf(x, 0.f), __fmul_rn(x, y)), log1pf(expf(-fabsf(x))));
}

// IOUloss(loss_type="iou"): 1 - iou^2, iou = area_i / (area_u + 1e-16)
__device__ __forceinline__ float yl_iou_loss(float px, float py, float pw, float ph, const YlGt& t) {
  const float tlx = fmaxf(px - pw / 2, t.cx - t.w / 2), tly = fmaxf(py - ph / 2, t.cy - t.h / 2);
  const float brx = fminf(px + pw / 2, t.cx + t.w / 2), bry = fminf(py + ph / 2, t.cy + t.h / 2);
  const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
  const float inter = (brx - tlx) * (bry - tly) * en;
  const float iou = inter / (pw * ph + t.w * t.h - inter + 1e-16f);
  return 1.f - iou * iou;
}

// minimum of one CTA per SM: without it ptxas caps the registers below what the loss terms need and spills
template <typename T>
__global__ void __launch_bounds__(YL_THREADS, 1)
yl_resolve_kernel(const T* __restrict__ outputs, const T* __restrict__ origin, const float* __restrict__ labels,
                  const float* __restrict__ shifts, int A, int C, int M, int use_l1, YlWs w) {
  __shared__ YlGt s_gt[YL_MAX_GT];
  __shared__ int s_n;
  __shared__ float s_red[4][YL_THREADS];
  __shared__ int s_fg[YL_THREADS];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int n = yl_load_gts(labels, b, M, C, s_gt, &s_n, nullptr);
  const int a = blockIdx.x * YL_THREADS + tid;
  float t_iou = 0.f, t_obj = 0.f, t_cls = 0.f, t_l1 = 0.f;
  int fg = 0;
  if (a < A) {
    const size_t ba = (size_t)b * A + a;
    const T* row = outputs + ba * (5 + C);
    const int cnt = w.count[ba];
    int m = -1;
    float iou_t = 0.f;
    if (cnt > 0) {
      const YlAnchor an = yl_anchor(shifts, A, a);
      m = w.chooser[ba];
      if (cnt > 1) {   // the argmin of the cost column over all GTs, first index on ties
        const float cs = w.cls_sum[ba], so = yl_sigmoid(yl_f(row[4]));
        float best = INFINITY, iou, c0;
        for (int g = 0; g < n; ++g) {
          const float c = yl_pair_cost(s_gt[g], an, row, cs, so, &iou, &c0);
          if (c < best || g == 0) { best = c; m = g; }
        }
      }
      const YlGt& gt = s_gt[m];
      const float px = yl_f(row[0]), py = yl_f(row[1]), pw = yl_f(row[2]), ph = yl_f(row[3]);
      iou_t = yl_iou(gt, px, py, pw, ph);
      fg = 1;
      t_iou = yl_iou_loss(px, py, pw, ph, gt);
      for (int c = 0; c < C; ++c) t_cls += yl_bce_logits(yl_f(row[5 + c]), c == gt.cls ? iou_t : 0.f);
      if (use_l1) {
        const float st = shifts[2 * A + a];
        const T* o = origin + ba * 4;
        t_l1 = fabsf(yl_f(o[0]) - (gt.cx / st - shifts[a])) + fabsf(yl_f(o[1]) - (gt.cy / st - shifts[A + a])) +
               fabsf(yl_f(o[2]) - logf(gt.w / st + 1e-8f)) + fabsf(yl_f(o[3]) - logf(gt.h / st + 1e-8f));
      }
    }
    t_obj = yl_bce_logits(yl_f(row[4]), fg ? 1.f : 0.f);
    w.fg[ba] = fg;
    w.matched[ba] = m;
    w.iou_t[ba] = iou_t;
  }
  s_red[0][tid] = t_iou; s_red[1][tid] = t_obj; s_red[2][tid] = t_cls; s_red[3][tid] = t_l1; s_fg[tid] = fg;
  __syncthreads();
  for (int h = YL_THREADS / 2; h; h >>= 1) {
    if (tid < h) {
#pragma unroll
      for (int q = 0; q < 4; ++q) s_red[q][tid] += s_red[q][tid + h];
      s_fg[tid] += s_fg[tid + h];
    }
    __syncthreads();
  }
  if (tid == 0) {
    const size_t p = (size_t)b * gridDim.x + blockIdx.x;
#pragma unroll
    for (int q = 0; q < 4; ++q) w.partial[p * 4 + q] = s_red[q][0];
    w.partial_fg[p] = s_fg[0];
  }
}

// ---------------------------------------------------------------------------------------------------------- stage 4
__global__ void __launch_bounds__(YL_THREADS) yl_finalize_kernel(int B, int P, int use_l1, YlWs w) {
  __shared__ float s_red[4][YL_THREADS];
  __shared__ int s_fg[YL_THREADS];
  const int tid = threadIdx.x;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  int fg = 0;
  for (int p = tid; p < P; p += YL_THREADS) {
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] += w.partial[(size_t)p * 4 + q];
    fg += w.partial_fg[p];
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) s_red[q][tid] = acc[q];
  s_fg[tid] = fg;
  __syncthreads();
  for (int h = YL_THREADS / 2; h; h >>= 1) {
    if (tid < h) {
#pragma unroll
      for (int q = 0; q < 4; ++q) s_red[q][tid] += s_red[q][tid + h];
      s_fg[tid] += s_fg[tid + h];
    }
    __syncthreads();
  }
  if (tid == 0) {
    int n_gt = 0, err = 0;
    for (int b = 0; b < B; ++b) { n_gt += w.nlabel[b]; err |= w.err[b]; }
    const float num_fg = (float)max(s_fg[0], 1);
    w.result[0] = 5.0f * (s_red[0][0] / num_fg);
    w.result[1] = s_red[1][0] / num_fg;
    w.result[2] = s_red[2][0] / num_fg;
    w.result[3] = use_l1 ? s_red[3][0] / num_fg : 0.f;
    w.result[4] = num_fg;
    w.result[5] = num_fg / (float)max(n_gt, 1);
    w.result[6] = (float)err;
    w.result[7] = (float)s_fg[0];
  }
}

// ---------------------------------------------------------------------------------------------------------- stage 5
// d(1 - iou^2)/d(pred column col) of IOUloss, torch's rules: max / min split the gradient evenly at ties, the tl < br
// gate has none.  gi = upstream gradient of the row's loss.
__device__ float yl_iou_loss_grad(float gi, float px, float py, float pw, float ph, const YlGt& t, int col) {
  const float ax = px - pw / 2, bx = t.cx - t.w / 2, ay = py - ph / 2, by = t.cy - t.h / 2;
  const float cx = px + pw / 2, dx = t.cx + t.w / 2, cy = py + ph / 2, dy = t.cy + t.h / 2;
  const float tlx = fmaxf(ax, bx), tly = fmaxf(ay, by), brx = fminf(cx, dx), bry = fminf(cy, dy);
  const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
  const float wx = brx - tlx, wy = bry - tly;
  const float inter = wx * wy * en;
  const float den = pw * ph + t.w * t.h - inter + 1e-16f;
  const float iou = inter / den;
  const float g_iou = gi * (-2.f * iou);
  const float g_den = -g_iou * inter / (den * den);
  const float g_inter = g_iou / den - g_den;               // inter enters the numerator and (negated) the denominator
  const float g_wx = g_inter * wy * en, g_wy = g_inter * wx * en;
  // weight of the prediction's side in max(tl) / min(br)
  const float s_tlx = ax > bx ? 1.f : (ax == bx ? 0.5f : 0.f), s_tly = ay > by ? 1.f : (ay == by ? 0.5f : 0.f);
  const float s_brx = cx < dx ? 1.f : (cx == dx ? 0.5f : 0.f), s_bry = cy < dy ? 1.f : (cy == dy ? 0.5f : 0.f);
  switch (col) {
    case 0: return g_wx * s_brx - g_wx * s_tlx;
    case 1: return g_wy * s_bry - g_wy * s_tly;
    case 2: return g_den * ph + 0.5f * (g_wx * s_brx + g_wx * s_tlx);
    default: return g_den * pw + 0.5f * (g_wy * s_bry + g_wy * s_tly);
  }
}

template <typename T>
__global__ void __launch_bounds__(YL_THREADS)
yl_backward_kernel(const T* __restrict__ outputs, const T* __restrict__ origin, const float* __restrict__ labels,
                   const float* __restrict__ shifts, int B, int A, int C, int M, int use_l1,
                   const float* __restrict__ grad_losses, YlWs w, T* __restrict__ grad_out, T* __restrict__ grad_origin) {
  const int D = 5 + C;
  const size_t n_out = (size_t)B * A * D, n_all = n_out + (use_l1 ? (size_t)B * A * 4 : 0);
  const size_t e = (size_t)blockIdx.x * YL_THREADS + threadIdx.x;
  if (e >= n_all) return;
  const float num_fg = w.result[4];
  if (e >= n_out) {   // origin_preds: L1 rows of fg anchors, sign(pred - target) with sign(0) = 0
    const size_t ba = (e - n_out) / 4;
    const int col = (int)((e - n_out) % 4), a = (int)(ba % A), b = (int)(ba / A);
    float g = 0.f;
    if (w.fg[ba]) {
      const float* L = labels + ((size_t)b * M + w.matched[ba]) * 5;
      const float st = shifts[2 * A + a];
      const float tgt = col == 0 ? L[1] / st - shifts[a] : col == 1 ? L[2] / st - shifts[A + a]
                                                                  : logf(L[1 + col] / st + 1e-8f);
      const float d = yl_f(origin[ba * 4 + col]) - tgt;
      g = (grad_losses[3] / num_fg) * (float)((d > 0.f) - (d < 0.f));
    }
    grad_origin[ba * 4 + col] = yl_to<T>(g);
    return;
  }
  const size_t ba = e / D;
  const int col = (int)(e % D), b = (int)(ba / A);
  const T* row = outputs + ba * D;
  const int fg = w.fg[ba];
  float g = 0.f;
  if (col == 4) {
    g = (grad_losses[1] / num_fg) * (yl_sigmoid(yl_f(row[4])) - (fg ? 1.f : 0.f));
  } else if (fg) {
    const float* L = labels + ((size_t)b * M + w.matched[ba]) * 5;
    const float cl = truncf(L[0]);
    const YlGt gt{L[1], L[2], L[3], L[4], (cl >= 0.f && cl < (float)C) ? (int)cl : 0};
    if (col < 4) {
      g = yl_iou_loss_grad((grad_losses[0] * 5.0f) / num_fg, yl_f(row[0]), yl_f(row[1]), yl_f(row[2]), yl_f(row[3]), gt,
                           col);
    } else {
      const float tgt = col - 5 == gt.cls ? w.iou_t[ba] : 0.f;
      g = (grad_losses[2] / num_fg) * (yl_sigmoid(yl_f(row[col])) - tgt);
    }
  }
  grad_out[e] = yl_to<T>(g);
}

template <typename T>
int yl_forward(const void* outputs, const void* origin, const float* labels, const float* shifts, int B, int A, int C, int M,
               int use_l1, float* trace, const YlWs& w, cudaStream_t st) {
  const T* o = static_cast<const T*>(outputs);
  const T* org = static_cast<const T*>(origin);
  const int nb = yl_blocks(A);
  yl_candidate_kernel<T><<<dim3(nb, B), YL_THREADS, 0, st>>>(o, labels, shifts, A, C, M, w);
  if (M > 0) yl_select_kernel<T><<<dim3(M, B), YL_THREADS, 0, st>>>(o, labels, shifts, A, C, M, trace, w);
  yl_resolve_kernel<T><<<dim3(nb, B), YL_THREADS, 0, st>>>(o, org, labels, shifts, A, C, M, use_l1, w);
  yl_finalize_kernel<<<1, YL_THREADS, 0, st>>>(B, B * nb, use_l1, w);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(M > 0 ? 4 : 3);
  return GDRN_OK;
}

template <typename T>
int yl_backward(const void* outputs, const void* origin, const float* labels, const float* shifts, int B, int A, int C, int M,
                int use_l1, const float* grad_losses, const YlWs& w, void* grad_out, void* grad_origin, cudaStream_t st) {
  const size_t n = (size_t)B * A * (5 + C) + (use_l1 ? (size_t)B * A * 4 : 0);
  yl_backward_kernel<T><<<(unsigned)((n + YL_THREADS - 1) / YL_THREADS), YL_THREADS, 0, st>>>(
      static_cast<const T*>(outputs), static_cast<const T*>(origin), labels, shifts, B, A, C, M, use_l1, grad_losses, w,
      static_cast<T*>(grad_out), static_cast<T*>(grad_origin));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

}  // namespace

extern "C" size_t yolox_loss_workspace_bytes(int B, int A, int M) {
  if (B <= 0 || A <= 0 || M < 0) return 0;
  return yl_layout(B, A, M).off[YL_NOFF] + 256;
}

extern "C" int yolox_loss_layout(int B, int A, int M, size_t* offsets) {
  GDRN_REQUIRE(offsets && B > 0 && A > 0 && M >= 0, "yolox_loss_layout: bad arguments");
  const YlLayout l = yl_layout(B, A, M);
  for (int k = 0; k < YL_NOFF; ++k) offsets[k] = l.off[k];
  return GDRN_OK;
}

#define YL_CHECK_ARGS(fn)                                                                                               \
  GDRN_REQUIRE(outputs && labels && shifts && workspace, fn ": null argument");                                        \
  GDRN_REQUIRE(B > 0 && A > 0 && num_classes > 0 && M >= 0, fn ": empty problem");                                      \
  GDRN_REQUIRE(M <= YL_MAX_GT, fn ": more than 1024 label rows per image");                                            \
  GDRN_REQUIRE(!use_l1 || origin_preds, fn ": use_l1 needs origin_preds");                                              \
  GDRN_REQUIRE(dtype >= 0 && dtype <= 2, fn ": dtype must be 0 (f32), 1 (f16) or 2 (bf16)");                            \
  GDRN_REQUIRE(workspace_bytes >= yolox_loss_workspace_bytes(B, A, M), fn ": workspace too small")

extern "C" int yolox_loss_forward(const void* outputs, const void* origin_preds, int dtype, const float* labels,
                                  const float* shifts, int B, int A, int num_classes, int M, int use_l1, float* trace,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  YL_CHECK_ARGS("yolox_loss_forward");
  const YlWs w = yl_ws(workspace, B, A, M);
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case 0: return yl_forward<float>(outputs, origin_preds, labels, shifts, B, A, num_classes, M, use_l1, trace, w, st);
    case 1: return yl_forward<__half>(outputs, origin_preds, labels, shifts, B, A, num_classes, M, use_l1, trace, w, st);
    default:
      return yl_forward<__nv_bfloat16>(outputs, origin_preds, labels, shifts, B, A, num_classes, M, use_l1, trace, w, st);
  }
}

extern "C" int yolox_loss_backward(const void* outputs, const void* origin_preds, int dtype, const float* labels,
                                   const float* shifts, int B, int A, int num_classes, int M, int use_l1,
                                   const float* grad_losses, void* workspace, size_t workspace_bytes, void* grad_outputs,
                                   void* grad_origin, void* stream) {
  YL_CHECK_ARGS("yolox_loss_backward");
  GDRN_REQUIRE(grad_losses && grad_outputs && (!use_l1 || grad_origin), "yolox_loss_backward: null gradient argument");
  const YlWs w = yl_ws(workspace, B, A, M);
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case 0:
      return yl_backward<float>(outputs, origin_preds, labels, shifts, B, A, num_classes, M, use_l1, grad_losses, w,
                                grad_outputs, grad_origin, st);
    case 1:
      return yl_backward<__half>(outputs, origin_preds, labels, shifts, B, A, num_classes, M, use_l1, grad_losses, w,
                                 grad_outputs, grad_origin, st);
    default:
      return yl_backward<__nv_bfloat16>(outputs, origin_preds, labels, shifts, B, A, num_classes, M, use_l1, grad_losses,
                                        w, grad_outputs, grad_origin, st);
  }
}
