// Device-side PVNet RANSAC voting layer: the whole of ransac_voting_layer / ransac_voting_layer_v3
// (core/csrc/ransac_voting/ransac_voting_gpu.py:7-104, 123-218) for a batch of masks in a handful of launches, with no
// host loop and no device -> host synchronisation.
//
// What the reference driver does per image, and what happens here instead:
//   torch.nonzero(mask) + masked_select(vertex)         -> rv_compact_kernel: ordered (row-major) compaction of the
//       (a device -> host sync for the shape)               foreground pixels into coords / direct, tn stays on the device
//   idxs = random_(0, tn) ONCE, outside the loop (:48)  -> hash RNG modulo tn on the device (or caller-supplied idxs)
//   while True: generate_hypothesis(idxs); vote; sum;   -> ONE round: the reference re-uses the same idxs every round, so
//       max; `all_win_ratio < cur_win_ratio` update;        every round yields the same hypotheses and counts and the
//       confidence test with .item()-style syncs            strict `<` update never fires again -- round 1 IS the result
//                                                           (hyp_num / confidence / max_iter only decide when the loop stops)
//   voting_for_hypothesis(all_win_pts) -> inlier mask;  -> rv_refit_kernel: inlier test of the winner + normal equations
//       ATA / ATb with torch.matmul; b_inv; matmul           (double accumulation) + 2x2 solve per keypoint, one CTA each
// Hypotheses, counts and inlier sets use the bit-exact arithmetic of rv_math.cuh (identical to the reference's CUDA
// build); the final 2x2 least squares agrees with torch's fp32 matmul / solve to rounding.
#include "common.cuh"
#include "rv_math.cuh"

namespace {

constexpr int RL_THREADS = 1024;

__device__ __forceinline__ unsigned rl_hash(unsigned x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// one CTA per image: count the foreground, optionally subsample it to ~max_num (ransac_voting_gpu.py:34-38), and compact
// coords (x, y) / direct in row-major order -- the order torch.nonzero / masked_select produce.  The mask holds integer
// weights (int)m: a pixel of non-zero weight is foreground, and foreground_num -- which decides min_num, max_num and
// the keep probability -- is the sum of the weights, as torch.sum of the reference's byte mask is
__global__ void __launch_bounds__(RL_THREADS)
rv_compact_kernel(const float* __restrict__ mask, const float* __restrict__ vertex, int h, int w, int vn, int min_num,
                  int max_num, unsigned seed, float* __restrict__ coords, float* __restrict__ direct, int* __restrict__ tn_out) {
  const int bi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int npix = h * w;
  const float* m = mask + (size_t)bi * npix;
  const float* vtx = vertex + (size_t)bi * npix * vn * 2;
  float* co = coords + (size_t)bi * npix * 2;
  float* di = direct + (size_t)bi * npix * vn * 2;
  __shared__ int s_scan[RL_THREADS / 32 + 1];
  __shared__ long long s_wsum[RL_THREADS / 32];
  __shared__ long long s_total;
  __shared__ int s_base;
  // pass 1: foreground weight
  long long c = 0;
  for (int i = tid; i < npix; i += RL_THREADS) c += (int)m[i];
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) s_wsum[warp] = c;
  __syncthreads();
  if (tid == 0) {
    long long t = 0;
    for (int k = 0; k < RL_THREADS / 32; ++k) t += s_wsum[k];
    s_total = t;
    s_base = 0;
  }
  __syncthreads();
  const long long fg = s_total;
  if (fg < min_num) {   // "if too few points, just skip it": zeros come out of the refit kernel
    if (tid == 0) tn_out[bi] = 0;
    return;
  }
  const bool subsample = fg > max_num;
  const float keep_p = subsample ? (float)max_num / (float)fg : 1.0f;
  // pass 2: ordered compaction, chunks of RL_THREADS pixels
  for (int base = 0; base < npix; base += RL_THREADS) {
    const int i = base + tid;
    bool sel = i < npix && (int)m[i] != 0;
    if (sel && subsample) {
      const float u = (float)(rl_hash(seed ^ rl_hash((unsigned)bi * 0x9E3779B9u + (unsigned)i)) >> 8) * (1.0f / 16777216.0f);
      sel = u < keep_p;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) s_scan[warp] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
      int acc = s_base;
      for (int k = 0; k < RL_THREADS / 32; ++k) { const int cc = s_scan[k]; s_scan[k] = acc; acc += cc; }
      s_scan[RL_THREADS / 32] = acc;
    }
    __syncthreads();
    if (sel) {
      const int slot = s_scan[warp] + __popc(bal & ((1u << lane) - 1u));
      co[slot * 2] = (float)(i % w);          // coords[:, [1, 0]]: (x, y)
      co[slot * 2 + 1] = (float)(i / w);
      for (int k = 0; k < vn * 2; ++k) di[(size_t)slot * vn * 2 + k] = vtx[(size_t)i * vn * 2 + k];
    }
    __syncthreads();
    if (tid == 0) s_base = s_scan[RL_THREADS / 32];
    __syncthreads();
  }
  if (tid == 0) tn_out[bi] = s_base;
}

// hypotheses of every (image, hypothesis, keypoint): idxs supplied ([b,hn,vn,2], taken modulo tn) or drawn on the device
__global__ void rv_gen_batched_kernel(const float* __restrict__ direct, const float* __restrict__ coords,
                                      const int* __restrict__ tn_p, const int* __restrict__ idxs, unsigned seed, int npix,
                                      int vn, int hn, float* __restrict__ hypo) {
  const int bi = blockIdx.y;
  const int hvi = blockIdx.x * blockDim.x + threadIdx.x;
  if (hvi >= hn * vn) return;
  const int tn = tn_p[bi];
  float* out = hypo + ((size_t)bi * hn * vn + hvi) * 2;
  out[0] = 0.f; out[1] = 0.f;                  // at::zeros in the reference: degenerate pairs stay (0, 0)
  if (tn <= 0) return;
  const int vi = hvi % vn;
  int t0, t1;
  if (idxs) {
    t0 = (int)((unsigned)idxs[((size_t)bi * hn * vn + hvi) * 2] % (unsigned)tn);
    t1 = (int)((unsigned)idxs[((size_t)bi * hn * vn + hvi) * 2 + 1] % (unsigned)tn);
  } else {
    const unsigned s0 = rl_hash(seed ^ rl_hash((unsigned)(bi * hn * vn + hvi) * 2u + 0x632BE5ABu));
    t0 = (int)(s0 % (unsigned)tn);
    t1 = (int)(rl_hash(s0 + 0x9E3779B9u) % (unsigned)tn);
  }
  const float* di = direct + (size_t)bi * npix * vn * 2;
  const float* co = coords + (size_t)bi * npix * 2;
  float hx, hy;
  if (rv_hypothesis(di[(t0 * vn + vi) * 2], di[(t0 * vn + vi) * 2 + 1], di[(t1 * vn + vi) * 2], di[(t1 * vn + vi) * 2 + 1],
                    co[t0 * 2], co[t0 * 2 + 1], co[t1 * 2], co[t1 * 2 + 1], &hx, &hy)) {
    out[0] = hx; out[1] = hy;
  }
}

// fused vote + count, batched: grid (pixel tiles of the LARGEST possible image, hypothesis chunks, images); tn per image
constexpr int RL_TILE_T = 256, RL_H_CHUNK = 32;
// largest dynamic shared memory of a launch (vn <= 84); the kernel opts in to all of it once, whatever vn comes first
constexpr size_t RL_SMEM_MAX = 200 * 1024;
__global__ void __launch_bounds__(RL_TILE_T)
rv_count_batched_kernel(const float* __restrict__ direct, const float* __restrict__ coords, const int* __restrict__ tn_p,
                        const float* __restrict__ hypo, int npix, int vn, int hn, float thresh, int* __restrict__ counts) {
  extern __shared__ float sm[];
  const int bi = blockIdx.z;
  const int tn = tn_p[bi];
  const int t0 = blockIdx.x * RL_TILE_T;
  if (t0 >= tn) return;
  float* s_dir = sm;
  float* s_hyp = s_dir + RL_TILE_T * vn * 2;
  int* s_cnt = reinterpret_cast<int*>(s_hyp + RL_H_CHUNK * vn * 2);
  const int h0 = blockIdx.y * RL_H_CHUNK;
  const int nh = min(RL_H_CHUNK, hn - h0), nt = min(RL_TILE_T, tn - t0);
  const int tid = threadIdx.x;
  const float* di = direct + (size_t)bi * npix * vn * 2;
  const float* co = coords + (size_t)bi * npix * 2;
  const float* hy = hypo + (size_t)bi * hn * vn * 2;
  for (int i = tid; i < nt * vn * 2; i += RL_TILE_T) s_dir[i] = di[(size_t)t0 * vn * 2 + i];
  for (int i = tid; i < nh * vn * 2; i += RL_TILE_T) s_hyp[i] = hy[(size_t)h0 * vn * 2 + i];
  for (int i = tid; i < nh * vn; i += RL_TILE_T) s_cnt[i] = 0;
  __syncthreads();
  const bool active = tid < nt;
  float cx = 0.f, cy = 0.f;
  if (active) { cx = co[(t0 + tid) * 2]; cy = co[(t0 + tid) * 2 + 1]; }
  for (int v = 0; v < vn; ++v) {
    float nx = 0.f, ny = 0.f, norm1 = 0.f;
    if (active) {
      nx = s_dir[(tid * vn + v) * 2];
      ny = s_dir[(tid * vn + v) * 2 + 1];
      norm1 = __fsqrt_rn(__fmaf_rn(nx, nx, __fmul_rn(ny, ny)));
    }
    for (int h = 0; h < nh; ++h) {
      const float* hp = s_hyp + (h * vn + v) * 2;
      const bool in = active && vote<false>(nx, ny, norm1, cx, cy, hp[0], hp[1], 0.f, thresh);
      const unsigned mm = __ballot_sync(0xffffffffu, in);
      if ((tid & 31) == 0 && mm) atomicAdd(&s_cnt[h * vn + v], __popc(mm));
    }
  }
  __syncthreads();
  for (int i = tid; i < nh * vn; i += RL_TILE_T)
    if (s_cnt[i]) atomicAdd(&counts[(size_t)bi * hn * vn + h0 * vn + i], s_cnt[i]);
}

// one CTA per (keypoint, image): winner = arg-max of the counts over the hypotheses (lowest index on ties), then the
// inlier set of the winner and the least-squares intersection of the inliers' lines (ransac_voting_gpu.py:78-102)
__global__ void __launch_bounds__(256)
rv_refit_kernel(const float* __restrict__ direct, const float* __restrict__ coords, const int* __restrict__ tn_p,
                const float* __restrict__ hypo, const int* __restrict__ counts, int npix, int vn, int hn, float thresh,
                float* __restrict__ win_pts, unsigned char* __restrict__ inliers) {
  const int v = blockIdx.x, bi = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tn = tn_p[bi];
  float* out = win_pts + ((size_t)bi * vn + v) * 2;
  __shared__ int s_best_c[8], s_best_h[8];
  __shared__ double s_acc[8][5];
  __shared__ float s_win[2];
  if (tn <= 0) {   // too few foreground pixels: the reference appends zeros (:29-32)
    if (tid == 0) { out[0] = 0.f; out[1] = 0.f; }
    return;
  }
  int bc = -1, bh = 0;
  for (int h = tid; h < hn; h += 256) {
    const int c = counts[((size_t)bi * hn + h) * vn + v];
    if (c > bc) { bc = c; bh = h; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int oc = __shfl_xor_sync(0xffffffffu, bc, o), oh = __shfl_xor_sync(0xffffffffu, bh, o);
    if (oc > bc || (oc == bc && oh < bh)) { bc = oc; bh = oh; }
  }
  if (lane == 0) { s_best_c[warp] = bc; s_best_h[warp] = bh; }
  __syncthreads();
  if (tid == 0) {
    int c = s_best_c[0], hh = s_best_h[0];
    for (int k = 1; k < 8; ++k)
      if (s_best_c[k] > c || (s_best_c[k] == c && s_best_h[k] < hh)) { c = s_best_c[k]; hh = s_best_h[k]; }
    // all_win_ratio starts at 0 and is replaced only by a strictly larger ratio: a winner with zero votes keeps (0, 0)
    const float* hp = hypo + (((size_t)bi * hn + hh) * vn + v) * 2;
    s_win[0] = c > 0 ? hp[0] : 0.f;
    s_win[1] = c > 0 ? hp[1] : 0.f;
  }
  __syncthreads();
  const float hx = s_win[0], hy = s_win[1];
  const float* di = direct + (size_t)bi * npix * vn * 2;
  const float* co = coords + (size_t)bi * npix * 2;
  double a00 = 0, a01 = 0, a11 = 0, b0 = 0, b1 = 0;
  for (int t = tid; t < tn; t += 256) {
    const float dx = di[((size_t)t * vn + v) * 2], dy = di[((size_t)t * vn + v) * 2 + 1];
    const float cx = co[t * 2], cy = co[t * 2 + 1];
    const float norm1 = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    const bool in = vote<false>(dx, dy, norm1, cx, cy, hx, hy, 0.f, thresh);
    if (inliers) inliers[((size_t)bi * vn + v) * npix + t] = in ? 1 : 0;
    if (in) {
      const double nx = (double)dy, ny = -(double)dx;          // normal = (d.y, -d.x)
      const double bb = nx * (double)cx + ny * (double)cy;
      a00 += nx * nx; a01 += nx * ny; a11 += ny * ny; b0 += nx * bb; b1 += ny * bb;
    }
  }
  double acc[5] = {a00, a01, a11, b0, b1};
  for (int k = 0; k < 5; ++k)
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  if (lane == 0) for (int k = 0; k < 5; ++k) s_acc[warp][k] = acc[k];
  __syncthreads();
  if (tid == 0) {
    double t[5] = {0, 0, 0, 0, 0};
    for (int w2 = 0; w2 < 8; ++w2) for (int k = 0; k < 5; ++k) t[k] += s_acc[w2][k];
    const double det = t[0] * t[2] - t[1] * t[1];
    double x, y;
    if (fabs(det) > 1e-12 * fmax(1.0, fabs(t[0] * t[2]))) {
      x = (t[2] * t[3] - t[1] * t[4]) / det;
      y = (t[0] * t[4] - t[1] * t[3]) / det;
    } else {   // singular ATA: the reference's b_inv falls back to the identity (ransac_voting_gpu.py:107-119)
      x = t[3]; y = t[4];
    }
    out[0] = (float)x; out[1] = (float)y;
  }
}

}  // namespace

extern "C" size_t rv_layer_workspace_bytes(int b, int h, int w, int vn, int hn) {
  if (b <= 0 || h <= 0 || w <= 0 || vn <= 0 || hn <= 0) return 0;
  const size_t npix = (size_t)h * w;
  return (size_t)b * npix * 2 * 4 + (size_t)b * npix * vn * 2 * 4 + (size_t)b * 4 + (size_t)b * hn * vn * 2 * 4 + (size_t)b * hn * vn * 4 + 1024;
}

extern "C" int rv_ransac_voting_layer(const float* mask, const float* vertex, int b, int h, int w, int vn, int hn,
                                      float inlier_thresh, int min_num, int max_num, unsigned seed, const int* idxs,
                                      float* win_pts, float* hypo_out, int* counts_out, int* tn_out, unsigned char* inliers,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(mask && vertex && win_pts && workspace, "ransac_voting_layer: null argument");
  GDRN_REQUIRE(b > 0 && h > 0 && w > 0 && vn > 0 && hn > 0, "ransac_voting_layer: empty problem");
  GDRN_REQUIRE(workspace_bytes >= rv_layer_workspace_bytes(b, h, w, vn, hn), "ransac_voting_layer: workspace too small");
  const size_t smem = (size_t)RL_TILE_T * vn * 8 + (size_t)RL_H_CHUNK * vn * 8 + (size_t)RL_H_CHUNK * vn * 4;
  GDRN_REQUIRE(smem <= RL_SMEM_MAX, "ransac_voting_layer: vn too large for the shared-memory tile");
  cudaStream_t st = (cudaStream_t)stream;
  const int npix = h * w;
  uint8_t* p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  float* coords = reinterpret_cast<float*>(p); p += (size_t)b * npix * 2 * 4;
  float* direct = reinterpret_cast<float*>(p); p += (size_t)b * npix * vn * 2 * 4;
  int* tn = reinterpret_cast<int*>(p); p += (((size_t)b * 4 + 255) / 256) * 256;
  float* hypo = hypo_out ? hypo_out : reinterpret_cast<float*>(p); p += (size_t)b * hn * vn * 2 * 4;
  int* counts = counts_out ? counts_out : reinterpret_cast<int*>(p);
  rv_compact_kernel<<<b, RL_THREADS, 0, st>>>(mask, vertex, h, w, vn, min_num, max_num, seed, coords, direct, tn);
  rv_gen_batched_kernel<<<dim3((hn * vn + 255) / 256, b), 256, 0, st>>>(direct, coords, tn, idxs, seed, npix, vn, hn, hypo);
  GDRN_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)b * hn * vn * 4, st));
  if (smem > 48 * 1024) GDRN_OPT_IN_SMEM(rv_count_batched_kernel, RL_SMEM_MAX);
  rv_count_batched_kernel<<<dim3((npix + RL_TILE_T - 1) / RL_TILE_T, (hn + RL_H_CHUNK - 1) / RL_H_CHUNK, b), RL_TILE_T, smem, st>>>(
      direct, coords, tn, hypo, npix, vn, hn, inlier_thresh, counts);
  rv_refit_kernel<<<dim3(vn, b), 256, 0, st>>>(direct, coords, tn, hypo, counts, npix, vn, hn, inlier_thresh, win_pts, inliers);
  if (tn_out) GDRN_CHECK_CUDA(cudaMemcpyAsync(tn_out, tn, (size_t)b * 4, cudaMemcpyDeviceToDevice, st));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(4);
  return GDRN_OK;
}
