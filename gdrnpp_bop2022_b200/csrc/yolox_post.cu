// YOLOX detection head post-processing on the GPU (SURVEY.md 8f rank 4): box decode, confidence filter, class-aware NMS.
//
// Replaces, for the detector stage in front of the pose path (det/yolox, demo/predictor_yolo.py):
//   YOLOXHead.decode_outputs            det/yolox/models/yolo_head.py:239-255   xy = (xy + grid) * stride, wh = exp(wh) * stride
//   postprocess(det_preds, num_classes, conf_thre, nms_thre, class_agnostic)    det/yolox/utils/boxes.py:34-80
//       cxcywh -> xyxy; class_conf, class_pred = max over the class scores; keep obj * class_conf >= conf_thre;
//       torchvision.ops.batched_nms / nms (greedy, IoU > nms_thre suppresses); rows (x1, y1, x2, y2, obj, cls_conf, cls)
// Per image, all on the device with no host synchronisation:
//   1. yolox_decode_filter_kernel: decode + filter + ORDERED compaction of the survivors (the order boolean indexing gives),
//      and the largest coordinate of the survivors (batched_nms' boxes.max())
//   2. yolox_rank_kernel: rank by descending score (ties: lower candidate index first) by counting -- candidates are few
//      hundred in practice, so an O(n^2) count beats a general sort and is deterministic
//   3. yolox_nms_mask_kernel: 64 x 64 IoU tiles -> suppression bit masks, with the decisions of torchvision on CUDA:
//      - class-aware, n <= 25 000 candidates (boxes.numel() <= 100 000): _batched_nms_coordinate_trick.  Every box is
//        shifted by cls * (max_coordinate + 1) in fp32 and every pair is compared, with no class check (the shift rounds
//        the coordinates, and with negative coordinates boxes of different classes can overlap and suppress);
//      - class-aware above 25 000 candidates: _batched_nms_vanilla, one NMS per class on the unshifted boxes;
//      - class-agnostic: nms on the unshifted boxes.
//      The IoU is the sm_90 build of torchvision's nms_kernel_impl<float>: the later-ranked box's area fused into the
//      denominator, fma(bw, bh, Sa) - inter, and IoU > (float)nms_thre.
//   4. yolox_nms_reduce_kernel: one warp walks the sorted candidates, ORs the masks of the kept ones, writes the kept rows
//      (the kept order is the rank order: the vanilla path's final score sort gives the same order when scores differ)
// The YOLOX network itself (backbone / PAFPN / head convolutions) runs in yolox_net.cu.
#include "common.cuh"

namespace {

constexpr int YX_THREADS = 1024;

__global__ void __launch_bounds__(YX_THREADS)
yolox_decode_filter_kernel(const float* __restrict__ preds, const int* __restrict__ hw, const int* __restrict__ strides, int n_levels,
                           int A, int nc, int decode, float conf_thre, float* __restrict__ cand /*[B,A,7]*/,
                           float* __restrict__ cand_score /*[B,A]*/, int* __restrict__ n_cand /*[B]*/,
                           float* __restrict__ max_coord /*[B]*/) {
  const int bi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = 5 + nc;
  const float* P = preds + (size_t)bi * A * C;
  float* out = cand + (size_t)bi * A * 7;
  float* outs = cand_score + (size_t)bi * A;
  __shared__ int s_scan[YX_THREADS / 32 + 1];
  __shared__ float s_wmax[YX_THREADS / 32];
  __shared__ int s_base;
  __shared__ float s_max;
  if (tid == 0) { s_base = 0; s_max = -INFINITY; }
  __syncthreads();
  for (int base = 0; base < A; base += YX_THREADS) {
    const int a = base + tid;
    bool keep = false;
    float row[7];
    float score = 0.f;
    if (a < A) {
      float cx = P[(size_t)a * C], cy = P[(size_t)a * C + 1], w = P[(size_t)a * C + 2], h = P[(size_t)a * C + 3];
      if (decode) {   // which pyramid level does anchor a belong to (levels are concatenated in order)
        int off = 0, lv = 0;
        for (; lv < n_levels; ++lv) {
          const int cnt = hw[lv * 2] * hw[lv * 2 + 1];
          if (a < off + cnt) break;
          off += cnt;
        }
        const int ww = hw[lv * 2 + 1];
        const float st = (float)strides[lv];
        const int loc = a - off;
        cx = __fmul_rn(__fadd_rn(cx, (float)(loc % ww)), st);
        cy = __fmul_rn(__fadd_rn(cy, (float)(loc / ww)), st);
        w = __fmul_rn(expf(w), st);
        h = __fmul_rn(expf(h), st);
      }
      const float hw2 = __fdiv_rn(w, 2.f), hh2 = __fdiv_rn(h, 2.f);
      row[0] = __fsub_rn(cx, hw2); row[1] = __fsub_rn(cy, hh2); row[2] = __fadd_rn(cx, hw2); row[3] = __fadd_rn(cy, hh2);
      const float obj = P[(size_t)a * C + 4];
      float best = -INFINITY;
      int bc = 0;
      for (int c = 0; c < nc; ++c) {
        const float v = P[(size_t)a * C + 5 + c];
        if (v > best) { best = v; bc = c; }   // first maximum, like torch.max
      }
      row[4] = obj; row[5] = best; row[6] = (float)bc;
      score = __fmul_rn(obj, best);
      keep = score >= conf_thre;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    float mx = keep ? fmaxf(fmaxf(row[0], row[1]), fmaxf(row[2], row[3])) : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) { s_scan[warp] = __popc(bal); s_wmax[warp] = mx; }
    __syncthreads();
    if (tid == 0) {
      int acc = s_base;
      for (int k = 0; k < YX_THREADS / 32; ++k) { const int c = s_scan[k]; s_scan[k] = acc; acc += c; }
      s_scan[YX_THREADS / 32] = acc;
      float m = s_max;
      for (int k = 0; k < YX_THREADS / 32; ++k) m = fmaxf(m, s_wmax[k]);
      s_max = m;
    }
    __syncthreads();
    if (keep) {
      const int slot = s_scan[warp] + __popc(bal & ((1u << lane) - 1u));
#pragma unroll
      for (int k = 0; k < 7; ++k) out[(size_t)slot * 7 + k] = row[k];
      outs[slot] = score;
    }
    __syncthreads();
    if (tid == 0) s_base = s_scan[YX_THREADS / 32];
    __syncthreads();
  }
  if (tid == 0) { n_cand[bi] = s_base; max_coord[bi] = s_max; }
}

// order[rank] = candidate index, rank by (score descending, index ascending)
__global__ void yolox_rank_kernel(const float* __restrict__ cand_score, const int* __restrict__ n_cand, int A, int* __restrict__ order) {
  const int bi = blockIdx.y;
  const int n = n_cand[bi];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = cand_score + (size_t)bi * A;
  const float si = s[i];
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const float sj = s[j];
    rank += (sj > si || (sj == si && j < i)) ? 1 : 0;
  }
  order[(size_t)bi * A + rank] = i;
}

// torchvision's nms_kernel_impl<float> as built for sm_90: a is the earlier-ranked box, b the later one, whose area is
// fused into the denominator (FFMA), so the denominator is rounded twice, not three times
__device__ __forceinline__ float yolox_iou(const float* a, const float* b) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float width = fmaxf(__fsub_rn(right, left), 0.f), height = fmaxf(__fsub_rn(bottom, top), 0.f);
  const float inter = __fmul_rn(width, height);
  const float Sa = __fmul_rn(__fsub_rn(a[2], a[0]), __fsub_rn(a[3], a[1]));
  return __fdiv_rn(inter, __fsub_rn(__fmaf_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]), Sa), inter));
}

constexpr int YX_TRICK_MAX_CAND = 25000;   // batched_nms on CUDA: coordinate trick while boxes.numel() <= 100 000

// mask[bi][i][jb] bit j set: sorted candidate (jb*64 + j) > i is suppressed by sorted candidate i.  The path (coordinate
// trick, vanilla or agnostic, see the header) is chosen per image from n_cand on the device.
__global__ void __launch_bounds__(64)
yolox_nms_mask_kernel(const float* __restrict__ cand, const int* __restrict__ order, const int* __restrict__ n_cand,
                      const float* __restrict__ max_coord, int A, int words, float nms_thre, int class_agnostic,
                      unsigned long long* __restrict__ mask) {
  const int bi = blockIdx.z;
  const int n = n_cand[bi];
  const int ib = blockIdx.y, jb = blockIdx.x;
  if (ib * 64 >= n || jb * 64 >= n || jb < ib) return;
  const bool trick = !class_agnostic && n <= YX_TRICK_MAX_CAND;
  const bool class_skip = !class_agnostic && !trick;
  const float step = trick ? __fadd_rn(max_coord[bi], 1.f) : 0.f;   // offsets = idxs * (max_coordinate + 1)
  __shared__ float sb[64][5];
  const int tid = threadIdx.x;
  const float* C = cand + (size_t)bi * A * 7;
  const int* ord = order + (size_t)bi * A;
  const int j = jb * 64 + tid;
  if (j < n) {
    const float* r = C + (size_t)ord[j] * 7;
    const float off = trick ? __fmul_rn(r[6], step) : 0.f;
    sb[tid][0] = __fadd_rn(r[0], off); sb[tid][1] = __fadd_rn(r[1], off);
    sb[tid][2] = __fadd_rn(r[2], off); sb[tid][3] = __fadd_rn(r[3], off); sb[tid][4] = r[6];
  }
  __syncthreads();
  const int i = ib * 64 + tid;
  if (i >= n) return;
  const float* ri = C + (size_t)ord[i] * 7;
  const float ci = ri[6];
  const float off = trick ? __fmul_rn(ci, step) : 0.f;
  const float a[4] = {__fadd_rn(ri[0], off), __fadd_rn(ri[1], off), __fadd_rn(ri[2], off), __fadd_rn(ri[3], off)};
  unsigned long long bits = 0;
  const int jn = min(64, n - jb * 64);
  for (int k = (ib == jb) ? tid + 1 : 0; k < jn; ++k) {
    if (class_skip && sb[k][4] != ci) continue;
    if (yolox_iou(a, sb[k]) > nms_thre) bits |= 1ull << k;
  }
  mask[((size_t)bi * A + i) * words + jb] = bits;
}

// one warp per image: greedy pass over the sorted candidates; the removed-set bit vector lives in shared memory
constexpr int YX_MAX_WORDS = 1024;   // up to 65 536 anchors per image
__global__ void __launch_bounds__(32)
yolox_nms_reduce_kernel(const float* __restrict__ cand, const int* __restrict__ order, const int* __restrict__ n_cand, int A, int words,
                        const unsigned long long* __restrict__ mask, int max_out, float* __restrict__ dets /*[B,max_out,7]*/,
                        int* __restrict__ n_det /*[B]*/) {
  __shared__ unsigned long long rem[YX_MAX_WORDS];
  const int bi = blockIdx.x, lane = threadIdx.x;
  const int n = n_cand[bi];
  const int nw = (n + 63) / 64;
  for (int w = lane; w < nw; w += 32) rem[w] = 0ull;
  __syncwarp();
  int kept = 0;
  const float* C = cand + (size_t)bi * A * 7;
  const int* ord = order + (size_t)bi * A;
  for (int i = 0; i < n; ++i) {
    const unsigned long long r = rem[i >> 6];      // warp-uniform read (writes are separated by __syncwarp)
    if ((r >> (i & 63)) & 1ull) continue;
    if (kept < max_out && lane < 7) dets[((size_t)bi * max_out + kept) * 7 + lane] = C[(size_t)ord[i] * 7 + lane];
    ++kept;
    const unsigned long long* mrow = mask + ((size_t)bi * A + i) * words;
    for (int w = (i >> 6) + lane; w < nw; w += 32) rem[w] |= mrow[w];
    __syncwarp();
  }
  if (lane == 0) n_det[bi] = kept < max_out ? kept : max_out;
}

// workspace layout, byte offsets from the 256-byte-aligned base: cand [B,A,7] f32, score [B,A] f32, order [B,A] i32,
// n_cand [B] i32, max_coord [B] f32, mask [B,A,words] u64
struct YxLayout {
  size_t off[6];
  size_t end;
};

YxLayout yx_layout(int B, int A) {
  const size_t words = (size_t)(A + 63) / 64;
  const size_t bytes[6] = {(size_t)B * A * 7 * 4, (size_t)B * A * 4, (size_t)B * A * 4, (size_t)B * 4, (size_t)B * 4,
                           (size_t)B * A * words * 8};
  YxLayout l;
  size_t p = 0;
  for (int k = 0; k < 6; ++k) { l.off[k] = p; p += (bytes[k] + 255) & ~(size_t)255; }
  l.end = p;
  return l;
}

}  // namespace

extern "C" size_t yolox_postprocess_workspace_bytes(int B, int A) {
  if (B <= 0 || A <= 0) return 0;
  return yx_layout(B, A).end + 256;
}

extern "C" int yolox_postprocess_layout(int B, int A, size_t* offsets) {
  GDRN_REQUIRE(offsets && B > 0 && A > 0, "yolox_postprocess_layout: bad arguments");
  const YxLayout l = yx_layout(B, A);
  for (int k = 0; k < 6; ++k) offsets[k] = l.off[k];
  return GDRN_OK;
}

extern "C" int yolox_postprocess(const float* preds, int B, int A, int num_classes, const int* hw, const int* strides, int n_levels,
                                 float conf_thre, float nms_thre, int class_agnostic, int max_out, float* dets, int* n_det,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(preds && dets && n_det && workspace, "yolox_postprocess: null argument");
  GDRN_REQUIRE(B > 0 && A > 0 && num_classes > 0 && max_out > 0, "yolox_postprocess: empty problem");
  GDRN_REQUIRE((A + 63) / 64 <= YX_MAX_WORDS, "yolox_postprocess: more than 65536 anchors per image");
  GDRN_REQUIRE(n_levels == 0 || (hw && strides), "yolox_postprocess: decode needs hw / strides (device int arrays)");
  GDRN_REQUIRE(workspace_bytes >= yolox_postprocess_workspace_bytes(B, A), "yolox_postprocess: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int words = (A + 63) / 64;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  const YxLayout l = yx_layout(B, A);
  float* cand = reinterpret_cast<float*>(base + l.off[0]);
  float* score = reinterpret_cast<float*>(base + l.off[1]);
  int* order = reinterpret_cast<int*>(base + l.off[2]);
  int* n_cand = reinterpret_cast<int*>(base + l.off[3]);
  float* max_coord = reinterpret_cast<float*>(base + l.off[4]);
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(base + l.off[5]);
  yolox_decode_filter_kernel<<<B, YX_THREADS, 0, st>>>(preds, hw, strides, n_levels, A, num_classes, n_levels > 0 ? 1 : 0, conf_thre, cand,
                                                       score, n_cand, max_coord);
  yolox_rank_kernel<<<dim3((A + 255) / 256, B), 256, 0, st>>>(score, n_cand, A, order);
  yolox_nms_mask_kernel<<<dim3(words, words, B), 64, 0, st>>>(cand, order, n_cand, max_coord, A, words, nms_thre, class_agnostic,
                                                              mask);
  yolox_nms_reduce_kernel<<<B, 32, 0, st>>>(cand, order, n_cand, A, words, mask, max_out, dets, n_det);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(4);
  return GDRN_OK;
}
