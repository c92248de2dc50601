// COCO bbox evaluation (pycocotools COCOeval.evaluate + accumulate, iouType "bbox", useCats) as four launches:
//
//   coco_match_kernel      one block per (image, category) pair: the stable descending score order of the pair's
//                          detections truncated to maxDets[-1], the IoU matrix (maskApi.c bbIou: no +1, float64, crowd GT
//                          divide by the detection area), the GT ignore flags per area range, and the greedy matching of
//                          evaluateImg for every (area range, IoU threshold): one thread each, GT visited non-ignored
//                          first (the stable sort on _ignore), threshold min(t, 1 - 1e-10), a matched GT skipped unless
//                          crowd, the break at the first ignored GT once a non-ignored match exists, and an unmatched
//                          detection outside the area range ignored.
//   coco_chunk_sort_kernel / coco_rank_kernel
//                          the per-category stable descending sort of accumulate (dtScores concatenated in image order,
//                          np.argsort(-s, kind="mergesort")): 1024-element chunks sorted in shared memory, then each
//                          element's rank is its rank in its chunk plus a binary search in every other chunk of its
//                          category.  Keys are (score descending, concatenation position ascending), a total order.
//   coco_accumulate_kernel one thread per (category, IoU threshold, area range, maxDets): cumulative TP / FP in float64,
//                          rc = tp / npig, pr = tp / (fp + tp + eps), the right-to-left precision envelope and
//                          searchsorted(rc, recThrs, "left") in one backward pass; -1 where the category has no pair or
//                          no non-ignored GT, 0 for recall thresholds past the last recall.
//
// Pairs are ordered by (category, image), so each category's GT and kept detections are contiguous.
#include "common.cuh"

namespace {

constexpr int kChunk = 1024;

__global__ void __launch_bounds__(128)
coco_match_kernel(const double* __restrict__ gt_box, const double* __restrict__ gt_area, const uint8_t* __restrict__ gt_crowd,
                  const double* __restrict__ dt_box, const double* __restrict__ dt_score, const int* __restrict__ pair_gt_off,
                  const int* __restrict__ pair_dt_off, const int* __restrict__ pair_kept_off, const long long* __restrict__ pair_iou_off,
                  int Gtot, int Dkept, const double* __restrict__ iou_thrs, int T, const double* __restrict__ area_rng, int A,
                  int max_det, int* __restrict__ dt_order, double* __restrict__ kept_score, int* __restrict__ kept_rank,
                  double* __restrict__ ious, uint8_t* __restrict__ gt_ignore, int* __restrict__ dt_match,
                  uint8_t* __restrict__ dt_ignore, int* __restrict__ gt_match) {
  const int p = blockIdx.x;
  const int g0 = pair_gt_off[p], G = pair_gt_off[p + 1] - g0;
  const int d0 = pair_dt_off[p], D = pair_dt_off[p + 1] - d0;
  const int k0 = pair_kept_off[p], Dk = pair_kept_off[p + 1] - k0;
  double* iou = ious + pair_iou_off[p];
  // stable descending order: rank = #(higher score) + #(equal score earlier)
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    const double s = dt_score[d0 + i];
    int r = 0;
    for (int j = 0; j < D; ++j) {
      const double o = dt_score[d0 + j];
      r += (o > s) || (o == s && j < i);
    }
    if (r < max_det) {
      dt_order[k0 + r] = d0 + i;
      kept_score[k0 + r] = s;
      kept_rank[k0 + r] = r;
    }
  }
  for (int i = threadIdx.x; i < A * G; i += blockDim.x) {
    const int a = i / G, g = i % G;
    const double ar = gt_area[g0 + g];
    gt_ignore[(long long)a * Gtot + g0 + g] = gt_crowd[g0 + g] || ar < area_rng[2 * a] || ar > area_rng[2 * a + 1];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Dk * G; i += blockDim.x) {
    const int r = i / G, g = i % G;
    const double* Dd = dt_box + 4 * (long long)dt_order[k0 + r];
    const double* Gg = gt_box + 4 * (long long)(g0 + g);
    const double da = __dmul_rn(Dd[2], Dd[3]), ga = __dmul_rn(Gg[2], Gg[3]);
    double o = 0.0;
    const double w = __dsub_rn(fmin(__dadd_rn(Dd[2], Dd[0]), __dadd_rn(Gg[2], Gg[0])), fmax(Dd[0], Gg[0]));
    if (w > 0) {
      const double h = __dsub_rn(fmin(__dadd_rn(Dd[3], Dd[1]), __dadd_rn(Gg[3], Gg[1])), fmax(Dd[1], Gg[1]));
      if (h > 0) {
        const double in = __dmul_rn(w, h);
        const double u = gt_crowd[g0 + g] ? da : __dsub_rn(__dadd_rn(da, ga), in);
        o = __ddiv_rn(in, u);
      }
    }
    iou[(long long)r * G + g] = o;
  }
  __syncthreads();
  if (threadIdx.x >= A * T) return;
  const int a = threadIdx.x / T, t = threadIdx.x % T;
  const long long row = (long long)(a * T + t);
  const uint8_t* gig = gt_ignore + (long long)a * Gtot + g0;
  int* gtm = gt_match + row * Gtot + g0;
  for (int g = 0; g < G; ++g) gtm[g] = 0;
  const double thr = fmin(iou_thrs[t], 1.0 - 1e-10);
  const double lo = area_rng[2 * a], hi = area_rng[2 * a + 1];
  for (int r = 0; r < Dk; ++r) {
    double best = thr;
    int m = -1;
    bool done = false;
    for (int pass = 0; pass < 2 && !done; ++pass) {
      for (int g = 0; g < G; ++g) {
        if (gig[g] != pass) continue;
        if (gtm[g] > 0 && !gt_crowd[g0 + g]) continue;
        if (m > -1 && gig[m] == 0 && pass == 1) { done = true; break; }
        const double v = iou[(long long)r * G + g];
        if (v < best) continue;
        best = v;
        m = g;
      }
    }
    const long long o = row * Dkept + k0 + r;
    if (m == -1) {
      const double* Dd = dt_box + 4 * (long long)dt_order[k0 + r];
      const double da = __dmul_rn(Dd[2], Dd[3]);
      dt_match[o] = 0;
      dt_ignore[o] = da < lo || da > hi;
    } else {
      dt_match[o] = g0 + m + 1;
      dt_ignore[o] = gig[m];
      gtm[m] = k0 + r + 1;
    }
  }
}

struct Key {
  double s;
  int pos;
};

__device__ __forceinline__ bool before(double sa, int pa, double sb, int pb) {   // a sorts before b
  return sa > sb || (sa == sb && pa < pb);
}

// grid (chunks, K): chunk c of category k sorted into sorted_s / sorted_p at the same positions
__global__ void __launch_bounds__(kChunk)
coco_chunk_sort_kernel(const double* __restrict__ score, const int* __restrict__ cat_off, double* __restrict__ sorted_s,
                       int* __restrict__ sorted_p) {
  __shared__ Key keys[kChunk];
  const int k = blockIdx.y;
  const int s0 = cat_off[k] + blockIdx.x * kChunk, s1 = min(cat_off[k + 1], s0 + kChunk);
  if (s0 >= s1) return;
  const int n = s1 - s0;
  const int i = threadIdx.x;
  if (i < n) keys[i] = {score[s0 + i], s0 + i};
  __syncthreads();
  if (i >= n) return;
  const Key me = keys[i];
  int r = 0;
  for (int j = 0; j < n; ++j) r += before(keys[j].s, keys[j].pos, me.s, me.pos);
  sorted_s[s0 + r] = me.s;
  sorted_p[s0 + r] = me.pos;
}

// grid (ceil(max n / 256), K): final position of every element of category k -> order[cat_off[k] + rank] = position
__global__ void __launch_bounds__(256)
coco_rank_kernel(const double* __restrict__ sorted_s, const int* __restrict__ sorted_p, const int* __restrict__ cat_off,
                 int* __restrict__ order) {
  const int k = blockIdx.y;
  const int c0 = cat_off[k], n = cat_off[k + 1] - c0;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double s = sorted_s[c0 + i];
  const int pos = sorted_p[c0 + i];
  const int mine = i / kChunk;
  int r = i - mine * kChunk;
  for (int c = 0; c * kChunk < n; ++c) {
    if (c == mine) continue;
    int lo = c * kChunk, hi = min(n, lo + kChunk);   // count of chunk c's keys that sort before (s, pos)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (before(sorted_s[c0 + mid], sorted_p[c0 + mid], s, pos)) lo = mid + 1;
      else hi = mid;
    }
    r += lo - c * kChunk;
  }
  order[c0 + r] = pos;
}

// one thread per (k, t, a, m); precision [T,R,K,A,M], recall [T,K,A,M] (both pre-filled with -1 by the host)
__global__ void __launch_bounds__(128)
coco_accumulate_kernel(const int* __restrict__ order, const int* __restrict__ cat_off, const int* __restrict__ cat_gt_off,
                       const int* __restrict__ cat_pairs, const int* __restrict__ kept_rank, const int* __restrict__ dt_match,
                       const uint8_t* __restrict__ dt_ignore, const uint8_t* __restrict__ gt_ignore, int Dkept, int Gtot,
                       int K, int T, int A, const double* __restrict__ rec_thrs, int R, const int* __restrict__ max_dets, int M,
                       double* __restrict__ precision, double* __restrict__ recall) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= K * T * A * M) return;
  const int m = idx % M, a = (idx / M) % A, t = (idx / (M * A)) % T, k = idx / (M * A * T);
  if (cat_pairs[k] == 0) return;   // no evaluateImg result for this category
  int npig = 0;
  for (int g = cat_gt_off[k]; g < cat_gt_off[k + 1]; ++g) npig += gt_ignore[(long long)a * Gtot + g] == 0;
  if (npig == 0) return;
  const int c0 = cat_off[k], n = cat_off[k + 1] - c0, maxd = max_dets[m];
  const long long row = (long long)(a * T + t) * Dkept;
  double tp = 0.0, fp = 0.0;
  int nd = 0;
  for (int i = 0; i < n; ++i) {
    const int pos = order[c0 + i];
    if (kept_rank[pos] >= maxd) continue;
    ++nd;
    if (dt_ignore[row + pos]) continue;
    if (dt_match[row + pos] != 0) tp += 1.0; else fp += 1.0;
  }
  const long long rk = ((long long)k * A + a) * M + m;   // recall [T,K,A,M], precision [T,R,K,A,M]
  const double np_d = (double)npig;
  recall[(long long)t * K * A * M + rk] = nd ? tp / np_d : 0.0;
  const double eps = 2.220446049250313e-16;   // np.spacing(1)
  int j = R - 1;
  double* q = precision + (long long)t * R * K * A * M + rk;
  const long long qstride = (long long)K * A * M;
  const double rc_last = tp / np_d;
  for (; j >= 0 && (nd == 0 || rec_thrs[j] > rc_last); --j) q[j * qstride] = 0.0;
  // Walking back over the kept detections, env is the envelope max(pr[i:]) of the element after the current one; the
  // thresholds in (rc[i], rc[i + 1]] have searchsorted index i + 1 and take that envelope.
  double env = 0.0;
  bool seen = false;
  for (int i = n - 1; i >= 0 && j >= 0; --i) {
    const int pos = order[c0 + i];
    if (kept_rank[pos] >= maxd) continue;
    const double rc = tp / np_d;
    const double pr = tp / __dadd_rn(__dadd_rn(fp, tp), eps);
    if (seen)
      for (; j >= 0 && rec_thrs[j] > rc; --j) q[j * qstride] = env;
    env = pr > env ? pr : env;
    seen = true;
    if (!dt_ignore[row + pos]) {
      if (dt_match[row + pos] != 0) tp -= 1.0; else fp -= 1.0;
    }
  }
  for (; seen && j >= 0; --j) q[j * qstride] = env;   // thresholds up to rc[0]: index 0
}

}  // namespace

extern "C" int coco_eval_match(const double* gt_box, const double* gt_area, const uint8_t* gt_crowd, const double* dt_box,
                               const double* dt_score, const int* pair_gt_off, const int* pair_dt_off, const int* pair_kept_off,
                               const long long* pair_iou_off, int P, int Gtot, int Dkept, const double* iou_thrs, int T,
                               const double* area_rng, int A, int max_det, int* dt_order, double* kept_score, int* kept_rank,
                               double* ious, uint8_t* gt_ignore, int* dt_match, uint8_t* dt_ignore, int* gt_match,
                               void* stream) {
  GDRN_REQUIRE(P >= 0 && Gtot >= 0 && Dkept >= 0 && T > 0 && A > 0 && A * T <= 128 && max_det > 0, "coco_eval_match: bad argument");
  if (P == 0) return GDRN_OK;
  GDRN_REQUIRE(pair_gt_off && pair_dt_off && pair_kept_off && pair_iou_off && iou_thrs && area_rng && kept_score && kept_rank &&
                   gt_ignore && dt_match && dt_ignore && gt_match && dt_order,
               "coco_eval_match: null argument");
  coco_match_kernel<<<P, 128, 0, (cudaStream_t)stream>>>(gt_box, gt_area, gt_crowd, dt_box, dt_score, pair_gt_off, pair_dt_off,
                                                         pair_kept_off, pair_iou_off, Gtot, Dkept, iou_thrs, T, area_rng, A,
                                                         max_det, dt_order, kept_score, kept_rank, ious, gt_ignore, dt_match,
                                                         dt_ignore, gt_match);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" size_t coco_eval_accumulate_workspace_bytes(int Dkept) {
  return (size_t)Dkept * (sizeof(double) + 2 * sizeof(int)) + 256;
}

extern "C" int coco_eval_accumulate(const double* kept_score, const int* kept_rank, const int* dt_match, const uint8_t* dt_ignore,
                                    const uint8_t* gt_ignore, const int* cat_off, const int* cat_gt_off, const int* cat_pairs,
                                    int max_cat_dets, int K, int Dkept, int Gtot, int T, int A, const double* rec_thrs, int R,
                                    const int* max_dets, int M, void* workspace, size_t workspace_bytes, double* precision,
                                    double* recall, void* stream) {
  GDRN_REQUIRE(K > 0 && Dkept >= 0 && Gtot >= 0 && T > 0 && A > 0 && R > 0 && M > 0 && max_cat_dets >= 0,
               "coco_eval_accumulate: bad argument");
  GDRN_REQUIRE(workspace_bytes >= coco_eval_accumulate_workspace_bytes(Dkept), "coco_eval_accumulate: workspace too small");
  GDRN_REQUIRE(cat_off && cat_gt_off && cat_pairs && rec_thrs && max_dets && precision && recall && workspace,
               "coco_eval_accumulate: null argument");
  const cudaStream_t s = (cudaStream_t)stream;
  double* sorted_s = (double*)workspace;
  int* sorted_p = (int*)(sorted_s + Dkept);
  int* order = sorted_p + Dkept;
  if (max_cat_dets > 0) {
    coco_chunk_sort_kernel<<<dim3((max_cat_dets + kChunk - 1) / kChunk, K), kChunk, 0, s>>>(kept_score, cat_off, sorted_s, sorted_p);
    GDRN_CHECK_CUDA(cudaGetLastError());
    coco_rank_kernel<<<dim3((max_cat_dets + 255) / 256, K), 256, 0, s>>>(sorted_s, sorted_p, cat_off, order);
    GDRN_CHECK_CUDA(cudaGetLastError());
  }
  const int threads = K * T * A * M;
  coco_accumulate_kernel<<<(threads + 127) / 128, 128, 0, s>>>(order, cat_off, cat_gt_off, cat_pairs, kept_rank, dt_match,
                                                               dt_ignore, gt_ignore, Dkept, Gtot, K, T, A, rec_thrs, R,
                                                               max_dets, M, precision, recall);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(max_cat_dets > 0 ? 3 : 1);
  return GDRN_OK;
}
