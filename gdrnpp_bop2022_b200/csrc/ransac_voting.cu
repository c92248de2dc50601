// PVNet vector-field RANSAC voting (hypothesis generation + inlier voting, plain and vanishing-point
// variants).  Replaces core/csrc/ransac_voting/src/ransac_voting_kernel.cu:11-49,88-126,170-229,268-310.
//
// Bit-exactness: the reference kernels are built by nvcc with the default --fmad=true, so WHICH products
// are fused is decided by ptxas.  The arithmetic below spells out, with explicit round-to-nearest
// intrinsics, the contraction ptxas 12.9 applies to the reference source for sm_90a (read from the SASS
// of the reference file compiled for sm_90a) so that hypotheses and inlier sets are bit-identical to the
// reference build on H100 (tests/golden/ref_cuda_golden.json).  sqrtf / __fdiv_rn are IEEE correctly rounded, as are
// sqrt.rn / div.rn in the reference.  The `< 1e-6` tests compare in double like the reference
// (1e-6 is a double literal, ransac_voting_kernel.cu:42-43,121).
//
// The voting kernel stages a tile of `direct`/`coords` (pixels) in shared memory once and sweeps all
// hypotheses over it: HBM traffic = 8*tn*vn + 8*tn + 8|12*hn*vn read, and either hn*vn*tn mask bytes
// written (reference-compatible entry) or 4*hn*vn count bytes (fused entry).
#include "common.cuh"
#include "rv_math.cuh"

namespace {

constexpr int RV_TILE_T = 256;
constexpr int RV_H_CHUNK = 32;

__global__ void gen_hyp_kernel(const float* __restrict__ direct, const float* __restrict__ coords,
                               const int* __restrict__ idxs, float* __restrict__ hypo, int tn, int vn, int hn) {
  int hvi = blockIdx.x * blockDim.x + threadIdx.x;
  if (hvi >= hn * vn) return;
  int vi = hvi % vn;
  int t0 = idxs[hvi * 2], t1 = idxs[hvi * 2 + 1];
  float d0x = direct[(t0 * vn + vi) * 2], d0y = direct[(t0 * vn + vi) * 2 + 1];
  float d1x = direct[(t1 * vn + vi) * 2], d1y = direct[(t1 * vn + vi) * 2 + 1];
  // normals n = (d.y, -d.x);  det_y = nx1*ny0 - nx0*ny1,  det_x = ny1*nx0 - ny0*nx1 = -det_y
  float a = __fmul_rn(d0x, d1y), b = __fmul_rn(d0y, d1x);
  float det_y = __fsub_rn(b, a);
  if ((double)fabsf(det_y) < 1e-6) return;
  float det_x = __fsub_rn(a, b);
  if ((double)fabsf(det_x) < 1e-6) return;
  float cx0 = coords[t0 * 2], cy0 = coords[t0 * 2 + 1];
  float cx1 = coords[t1 * 2], cy1 = coords[t1 * 2 + 1];
  float s1 = __fmaf_rn(d1y, cx1, -__fmul_rn(d1x, cy1));  // nx1*cx1 + ny1*cy1
  float s0 = __fmaf_rn(d0y, cx0, -__fmul_rn(d0x, cy0));  // nx0*cx0 + ny0*cy0
  float num_y = __fmaf_rn(d1y, s0, -__fmul_rn(d0y, s1));
  float num_x = __fmaf_rn(-d1x, s0, __fmul_rn(d0x, s1));
  hypo[hvi * 2] = __fdiv_rn(num_x, det_x);
  hypo[hvi * 2 + 1] = __fdiv_rn(num_y, det_y);
}

__global__ void gen_hyp_vp_kernel(const float* __restrict__ direct, const float* __restrict__ coords,
                                  const int* __restrict__ idxs, float* __restrict__ hypo, int tn, int vn, int hn) {
  int hvi = blockIdx.x * blockDim.x + threadIdx.x;
  if (hvi >= hn * vn) return;
  int vi = hvi % vn;
  int id0 = idxs[hvi * 2], id1 = idxs[hvi * 2 + 1];
  float dx0 = direct[(id0 * vn + vi) * 2], dy0 = direct[(id0 * vn + vi) * 2 + 1];
  float dx1 = direct[(id1 * vn + vi) * 2], dy1 = direct[(id1 * vn + vi) * 2 + 1];
  float cx0 = coords[id0 * 2], cy0 = coords[id0 * 2 + 1];
  float cx1 = coords[id1 * 2], cy1 = coords[id1 * 2 + 1];
  // lines l = (dy, -dx, cy*dx - cx*dy); (x,y,z) = l0 x l1
  float lz0 = __fmaf_rn(dx0, cy0, -__fmul_rn(dy0, cx0));
  float lz1 = __fmaf_rn(dx1, cy1, -__fmul_rn(dy1, cx1));
  float x = __fmaf_rn(dx1, lz0, -__fmul_rn(dx0, lz1));
  float y = __fmaf_rn(dy1, lz0, -__fmul_rn(dy0, lz1));
  float z = __fmaf_rn(dx0, dy1, -__fmul_rn(dy0, dx1));
  float vx0 = __fmul_rn(dx0, __fmaf_rn(-cx0, z, x));
  float vx1 = __fmul_rn(dx1, __fmaf_rn(-cx1, z, x));
  float vy0 = __fmul_rn(dy0, __fmaf_rn(-cy0, z, y));
  float vy1 = __fmul_rn(dy1, __fmaf_rn(-cy1, z, y));
  if (vx0 < 0 && vx1 < 0 && vy0 < 0 && vy1 < 0) { x = -x; y = -y; z = -z; }
  if (__fmul_rn(vx0, vx1) < 0 || __fmul_rn(vy0, vy1) < 0) { x = 0.f; y = 0.f; z = 0.f; }
  hypo[hvi * 3] = x;
  hypo[hvi * 3 + 1] = y;
  hypo[hvi * 3 + 2] = z;
}

// grid: (ceil(tn / RV_TILE_T), ceil(hn / RV_H_CHUNK)); block RV_TILE_T threads, one pixel per thread.
template <bool VP, bool COUNT>
__global__ void __launch_bounds__(RV_TILE_T)
vote_kernel(const float* __restrict__ direct, const float* __restrict__ coords, const float* __restrict__ hypo,
            unsigned char* __restrict__ inliers, int* __restrict__ counts, int tn, int vn, int hn, float thresh) {
  extern __shared__ float sm[];
  constexpr int HD = VP ? 3 : 2;
  float* s_dir = sm;                              // [RV_TILE_T][vn][2]
  float* s_hyp = s_dir + RV_TILE_T * vn * 2;      // [RV_H_CHUNK][vn][HD]
  int* s_cnt = reinterpret_cast<int*>(s_hyp + RV_H_CHUNK * vn * HD);  // [RV_H_CHUNK][vn]
  const int t0 = blockIdx.x * RV_TILE_T;
  const int h0 = blockIdx.y * RV_H_CHUNK;
  const int nh = min(RV_H_CHUNK, hn - h0);
  const int nt = min(RV_TILE_T, tn - t0);
  const int tid = threadIdx.x;
  for (int i = tid; i < nt * vn * 2; i += RV_TILE_T) s_dir[i] = direct[(size_t)t0 * vn * 2 + i];
  for (int i = tid; i < nh * vn * HD; i += RV_TILE_T) s_hyp[i] = hypo[(size_t)h0 * vn * HD + i];
  if (COUNT)
    for (int i = tid; i < nh * vn; i += RV_TILE_T) s_cnt[i] = 0;
  __syncthreads();
  const int t = t0 + tid;
  const bool active = tid < nt;
  float cx = 0.f, cy = 0.f;
  if (active) { cx = coords[t * 2]; cy = coords[t * 2 + 1]; }
  for (int v = 0; v < vn; ++v) {
    float nx = 0.f, ny = 0.f, norm1 = 0.f;
    if (active) {
      nx = s_dir[(tid * vn + v) * 2];
      ny = s_dir[(tid * vn + v) * 2 + 1];
      norm1 = __fsqrt_rn(__fmaf_rn(nx, nx, __fmul_rn(ny, ny)));
    }
    for (int h = 0; h < nh; ++h) {
      const float* hp = s_hyp + (h * vn + v) * HD;
      bool in = active && vote<VP>(nx, ny, norm1, cx, cy, hp[0], hp[1], VP ? hp[HD - 1] : 0.f, thresh);
      if (COUNT) {
        unsigned m = __ballot_sync(0xffffffffu, in);
        if ((tid & 31) == 0 && m) atomicAdd(&s_cnt[h * vn + v], __popc(m));
      } else if (in) {
        inliers[((size_t)(h0 + h) * vn + v) * tn + t] = 1;
      }
    }
  }
  if (COUNT) {
    __syncthreads();
    for (int i = tid; i < nh * vn; i += RV_TILE_T)
      if (s_cnt[i]) atomicAdd(&counts[h0 * vn + i], s_cnt[i]);
  }
}

template <bool VP, bool COUNT>
int vote_launch(const float* direct, const float* coords, const float* hypo, unsigned char* inliers, int* counts,
                int tn, int vn, int hn, float thresh, cudaStream_t st) {
  GDRN_REQUIRE(tn > 0 && vn > 0 && hn > 0, "ransac_voting: tn, vn, hn must be positive");
  size_t smem = (size_t)RV_TILE_T * vn * 8 + (size_t)RV_H_CHUNK * vn * (VP ? 12 : 8) + (size_t)RV_H_CHUNK * vn * 4;
  GDRN_REQUIRE(smem <= 200 * 1024, "ransac_voting: vn too large for the shared-memory tile");
  auto k = vote_kernel<VP, COUNT>;
  if (smem > 48 * 1024) GDRN_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((tn + RV_TILE_T - 1) / RV_TILE_T, (hn + RV_H_CHUNK - 1) / RV_H_CHUNK);
  if (COUNT) GDRN_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)hn * vn * 4, st));
  k<<<grid, RV_TILE_T, smem, st>>>(direct, coords, hypo, inliers, counts, tn, vn, hn, thresh);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

}  // namespace

extern "C" int rv_generate_hypothesis(const float* direct, const float* coords, const int* idxs, float* hypo, int tn,
                                      int vn, int hn, void* stream) {
  GDRN_REQUIRE(tn > 0 && vn > 0 && hn > 0, "ransac_voting: tn, vn, hn must be positive");
  int n = hn * vn;
  gen_hyp_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(direct, coords, idxs, hypo, tn, vn, hn);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
extern "C" int rv_generate_hypothesis_vanishing_point(const float* direct, const float* coords, const int* idxs,
                                                      float* hypo, int tn, int vn, int hn, void* stream) {
  GDRN_REQUIRE(tn > 0 && vn > 0 && hn > 0, "ransac_voting: tn, vn, hn must be positive");
  int n = hn * vn;
  gen_hyp_vp_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(direct, coords, idxs, hypo, tn, vn, hn);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
extern "C" int rv_voting_for_hypothesis(const float* direct, const float* coords, const float* hypo,
                                        unsigned char* inliers, int tn, int vn, int hn, float inlier_thresh,
                                        void* stream) {
  return vote_launch<false, false>(direct, coords, hypo, inliers, nullptr, tn, vn, hn, inlier_thresh,
                                   (cudaStream_t)stream);
}
extern "C" int rv_voting_for_hypothesis_vanishing_point(const float* direct, const float* coords, const float* hypo,
                                                        unsigned char* inliers, int tn, int vn, int hn,
                                                        float inlier_thresh, void* stream) {
  return vote_launch<true, false>(direct, coords, hypo, inliers, nullptr, tn, vn, hn, inlier_thresh,
                                  (cudaStream_t)stream);
}
extern "C" int rv_vote_count(const float* direct, const float* coords, const float* hypo, int* counts, int tn, int vn,
                             int hn, float inlier_thresh, int vanishing_point, void* stream) {
  if (vanishing_point)
    return vote_launch<true, true>(direct, coords, hypo, nullptr, counts, tn, vn, hn, inlier_thresh,
                                   (cudaStream_t)stream);
  return vote_launch<false, true>(direct, coords, hypo, nullptr, counts, tn, vn, hn, inlier_thresh,
                                  (cudaStream_t)stream);
}
