// BOP pose errors: VSD, MSSD / MSPD and ADD / ADI over a batch of (estimate, GT) pairs.
// Replaces the per-pair numpy loops of lib/pysixd/pose_error.py (vsd :22-128, mssd :131-153, mspd :156-179,
// add :256-271, adi :274-296) as driven by lib/pysixd/scripts/eval_calc_errors.py:345-475.
//
// Every result is independent of the launch shape:
//  * VSD is a set of integer pixel counts per pair (union, intersection, and per tau the pixels with cost 1), summed with
//    64-bit integer atomics; the error is formed from the counts in one rounding, as the reference forms it.
//  * MSSD / MSPD are a max over points and a min over symmetries of non-negative doubles, combined across CTAs with
//    atomicMax / atomicMin on the bit patterns (for non-negative IEEE doubles the order of the patterns is the order of
//    the values).
//  * ADD / ADI sum per-point distances in a fixed order: fixed 256-point chunks, a fixed in-CTA tree, then the chunk
//    partials in chunk order.
#include <math.h>

#include "bop_visib.cuh"
#include "common.cuh"

namespace {

constexpr int VSD_THREADS = 256;
constexpr int VSD_MAX_T = 32;
constexpr int SYM_BLOCK = 8;       // symmetries per CTA, one per warp
constexpr int SYM_THREADS = SYM_BLOCK * 32;
constexpr int AD_THREADS = 256;    // also the point chunk of one CTA
constexpr int AD_TILE = 512;       // estimate-pose points per shared-memory tile of the ADI search
constexpr int RT_THREADS = 128;    // sym_rt_kernel: 4 pairs per CTA, one warp each

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ unsigned warp_sum_u(unsigned v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// counts[p] = {union, intersection, cost(tau_0), ..., cost(tau_{T-1})}
__global__ void __launch_bounds__(VSD_THREADS)
vsd_count_kernel(const float* __restrict__ depth_est, const float* __restrict__ depth_gt, const float* __restrict__ depth_test,
                 int H, int W, const int* __restrict__ pair_est, const int* __restrict__ pair_gt,
                 const int* __restrict__ pair_img, const double* __restrict__ Ks, const double* __restrict__ diameters,
                 const uint8_t* __restrict__ gate, const double* __restrict__ taus, int T, float delta, int normalized,
                 unsigned long long* __restrict__ counts) {
  const int p = blockIdx.x;   // pairs on x (no 65535 cap), pixel slices on y
  if (!gate[p]) return;
  __shared__ double s_tau[VSD_MAX_T];
  __shared__ unsigned s_red[VSD_THREADS / 32][VSD_MAX_T + 2];
  if (threadIdx.x < T) s_tau[threadIdx.x] = taus[threadIdx.x];
  __syncthreads();
  const double* K = Ks + (size_t)p * 9;
  const double fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  const double diam = diameters[p];
  const size_t HW = (size_t)H * W;
  const float* de = depth_est + (size_t)pair_est[p] * HW;
  const float* dg = depth_gt + (size_t)pair_gt[p] * HW;
  const float* dt = depth_test + (size_t)pair_img[p] * HW;
  // union / intersection per thread; the cost count of tau k is kept by lane k from warp ballots (T <= 32), so the
  // register count does not grow with T.  The pixel loop has a warp-uniform trip count for the ballots.
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned n_union = 0, n_inter = 0, n_cost = 0;
  for (size_t base = (size_t)blockIdx.y * VSD_THREADS; base < HW; base += (size_t)gridDim.y * VSD_THREADS) {
    const size_t i = base + threadIdx.x;
    bool inter = false;
    double d = 0.0;
    const float ze = i < HW ? de[i] : 0.f, zg = i < HW ? dg[i] : 0.f;
    if (ze != 0.f || zg != 0.f) {   // else d_model > 0 fails in both masks: the pixel is in neither
      const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
      const double pre_x = __ddiv_rn(__dsub_rn((double)x, cx), fx);
      const double pre_y = __ddiv_rn(__dsub_rn((double)y, cy), fy);
      const double dist_e = dist_px(pre_x, pre_y, ze), dist_g = dist_px(pre_x, pre_y, zg);
      const double dist_t = dist_px(pre_x, pre_y, dt[i]);
      const bool v_gt = visib_bop19(dist_g, dist_t, delta);
      const bool v_est = visib_bop19(dist_e, dist_t, delta) || (v_gt && dist_e > 0.0);   // estimate_visib_mask_est
      n_union += (v_gt || v_est);
      inter = v_gt && v_est;
      if (inter) {
        ++n_inter;
        d = fabs(__dsub_rn(dist_g, dist_e));
        if (normalized) d = __ddiv_rn(d, diam);
      }
    }
    if (__any_sync(0xffffffffu, inter)) {
      for (int k = 0; k < T; ++k) {
        const unsigned b = __ballot_sync(0xffffffffu, inter && d >= s_tau[k]);
        if (lane == k) n_cost += __popc(b);
      }
    }
  }
  n_union = warp_sum_u(n_union);
  n_inter = warp_sum_u(n_inter);
  if (lane == 0) { s_red[warp][0] = n_union; s_red[warp][1] = n_inter; }
  if (lane < T) s_red[warp][lane + 2] = n_cost;
  __syncthreads();
  if (threadIdx.x < T + 2) {
    unsigned long long s = 0;
    for (int w = 0; w < VSD_THREADS / 32; ++w) s += s_red[w][threadIdx.x];
    if (s) atomicAdd(counts + (size_t)p * (T + 2) + threadIdx.x, s);
  }
}

// pose_error.vsd :110-126: (sum(costs) + (union - inter)) / float(union), or 1.0 for an empty union; eval_calc_errors.py
// :376-378: 1.0 for every tau when the sphere projections do not overlap (gate 0).
__global__ void vsd_finalize_kernel(const unsigned long long* __restrict__ counts, const uint8_t* __restrict__ gate, int P,
                                    int T, double* __restrict__ errors) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P * T) return;
  const int p = i / T, k = i - p * T;
  const unsigned long long* c = counts + (size_t)p * (T + 2);
  if (!gate[p] || c[0] == 0) {
    errors[i] = 1.0;
    return;
  }
  errors[i] = __ddiv_rn((double)(long long)(c[k + 2] + (c[0] - c[1])), (double)(long long)c[0]);
}

// 3x4 pose [R|t] (row-major) applied to x
__device__ __forceinline__ void xform(const double* M, double x, double y, double z, double& ox, double& oy, double& oz) {
  ox = fma(M[0], x, fma(M[1], y, fma(M[2], z, M[3])));
  oy = fma(M[4], x, fma(M[5], y, fma(M[6], z, M[7])));
  oz = fma(M[8], x, fma(M[9], y, fma(M[10], z, M[11])));
}
// misc.project_pts (misc.py:568-582): P = K [R|t] applied to [x, 1], divided by the third row
__device__ __forceinline__ void project(const double* Pm, double x, double y, double z, double& u, double& v) {
  double a, b, c;
  xform(Pm, x, y, z, a, b, c);
  const double r = 1.0 / c;
  u = a * r;
  v = b * r;
}
// out = K [R|t] (3x3 times 3x4)
__device__ __forceinline__ void k_times(const double* K, const double* M, double* out) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) out[r * 4 + c] = K[r * 3] * M[c] + K[r * 3 + 1] * M[4 + c] + K[r * 3 + 2] * M[8 + c];
}

__global__ void sym_init_kernel(double* __restrict__ mssd, double* __restrict__ mspd, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) { mssd[i] = INFINITY; mspd[i] = INFINITY; }
}

// grid (P, ceil(max_syms / SYM_BLOCK)): one CTA = one pair x up to SYM_BLOCK symmetries of its object, all its points;
// warp w owns symmetry w of the block.  Points stream through shared memory in tiles; the estimate-pose point and its
// projection are computed once per tile and read by every warp.
__global__ void __launch_bounds__(SYM_THREADS)
sym_max_dist_kernel(const double* __restrict__ pts, const int64_t* __restrict__ pt_off, const double* __restrict__ syms,
                    const int64_t* __restrict__ sym_off, const int* __restrict__ pair_obj, const double* __restrict__ pose_est,
                    const double* __restrict__ pose_gt, const double* __restrict__ Ks, const uint8_t* __restrict__ gate_mssd,
                    double* __restrict__ mssd, double* __restrict__ mspd) {
  const int p = blockIdx.x, o = pair_obj[p];
  const int64_t s0 = sym_off[o] + (int64_t)blockIdx.y * SYM_BLOCK;
  const int ns = (int)min((int64_t)SYM_BLOCK, sym_off[o + 1] - s0);
  if (ns <= 0) return;
  const bool do_mssd = gate_mssd[p] != 0;
  __shared__ double s_est[12], s_pest[12], s_gs[SYM_BLOCK][12], s_pgs[SYM_BLOCK][12];
  __shared__ double s_tile[8][SYM_THREADS];   // x, y, z, estimate-pose x, y, z, projection u, v
  __shared__ double s_red[SYM_BLOCK][2];
  const double* K = Ks + (size_t)p * 9;
  const double* Pg = pose_gt + (size_t)p * 12;
  if (threadIdx.x == 0) {
    for (int j = 0; j < 12; ++j) s_est[j] = pose_est[(size_t)p * 12 + j];
    k_times(K, s_est, s_pest);
  }
  if (threadIdx.x < ns) {   // pose_error.mssd/mspd: R_gt_sym = R_gt . R_sym, t_gt_sym = R_gt . t_sym + t_gt
    const double* S = syms + (size_t)(s0 + threadIdx.x) * 12;
    double* G = s_gs[threadIdx.x];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) G[r * 4 + c] = Pg[r * 4] * S[c] + Pg[r * 4 + 1] * S[4 + c] + Pg[r * 4 + 2] * S[8 + c];
      G[r * 4 + 3] = (Pg[r * 4] * S[3] + Pg[r * 4 + 1] * S[7] + Pg[r * 4 + 2] * S[11]) + Pg[r * 4 + 3];
    }
    k_times(K, G, s_pgs[threadIdx.x]);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ws = min(warp, ns - 1);   // warps past ns idle in the point loop but keep the barriers
  double G[12], PG[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) { G[j] = s_gs[ws][j]; PG[j] = s_pgs[ws][j]; }
  double md = 0.0, mp = 0.0;   // max squared distance / squared pixel distance
  const double* X = pts + (size_t)pt_off[o] * 3;
  const int n = (int)(pt_off[o + 1] - pt_off[o]);
  for (int t0 = 0; t0 < n; t0 += SYM_THREADS) {
    const int cnt = min(SYM_THREADS, n - t0);
    __syncthreads();
    if (threadIdx.x < cnt) {
      const int i = t0 + threadIdx.x;
      const double x = X[i * 3], y = X[i * 3 + 1], z = X[i * 3 + 2];
      double ex, ey, ez, eu, ev;
      xform(s_est, x, y, z, ex, ey, ez);
      project(s_pest, x, y, z, eu, ev);
      s_tile[0][threadIdx.x] = x; s_tile[1][threadIdx.x] = y; s_tile[2][threadIdx.x] = z;
      s_tile[3][threadIdx.x] = ex; s_tile[4][threadIdx.x] = ey; s_tile[5][threadIdx.x] = ez;
      s_tile[6][threadIdx.x] = eu; s_tile[7][threadIdx.x] = ev;
    }
    __syncthreads();
    if (warp < ns) {
      for (int j = lane; j < cnt; j += 32) {
        const double x = s_tile[0][j], y = s_tile[1][j], z = s_tile[2][j];
        if (do_mssd) {
          double gx, gy, gz;
          xform(G, x, y, z, gx, gy, gz);
          const double dx = s_tile[3][j] - gx, dy = s_tile[4][j] - gy, dz = s_tile[5][j] - gz;
          md = fmax(md, dx * dx + dy * dy + dz * dz);
        }
        double gu, gv;
        project(PG, x, y, z, gu, gv);
        const double du = s_tile[6][j] - gu, dv = s_tile[7][j] - gv;
        mp = fmax(mp, du * du + dv * dv);
      }
    }
  }
  md = warp_max_d(md);
  mp = warp_max_d(mp);
  if (lane == 0 && warp < ns) { s_red[warp][0] = md; s_red[warp][1] = mp; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double best_d = INFINITY, best_p = INFINITY;
    for (int s = 0; s < ns; ++s) {   // sqrt is monotone: the root of the max is the max of the roots
      best_d = fmin(best_d, sqrt(s_red[s][0]));
      best_p = fmin(best_p, sqrt(s_red[s][1]));
    }
    if (do_mssd) atomicMin((unsigned long long*)(mssd + p), (unsigned long long)__double_as_longlong(best_d));
    atomicMin((unsigned long long*)(mspd + p), (unsigned long long)__double_as_longlong(best_p));
  }
}

__global__ void fill_inf_kernel(double* __restrict__ out, int P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) out[i] = INFINITY;
}

// The pose a pair is compared against: the GT pose composed with symmetry S (R_g . R_s, R_g . t_s + t_g), or the GT
// pose itself when S is null (proj / re / te: the identity is not always in an object's symmetry set, see
// misc.get_symmetry_transformations).
__device__ __forceinline__ void gt_sym_pose(const double* Pg, const double* S, double* G) {
  if (!S) {
    for (int j = 0; j < 12; ++j) G[j] = Pg[j];
    return;
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) G[r * 4 + c] = Pg[r * 4] * S[c] + Pg[r * 4 + 1] * S[4 + c] + Pg[r * 4 + 2] * S[8 + c];
    G[r * 4 + 3] = (Pg[r * 4] * S[3] + Pg[r * 4 + 1] * S[7] + Pg[r * 4 + 2] * S[11]) + Pg[r * 4 + 3];
  }
}

// misc.transform_pts_Rt_2d (pose_error.py:236-253): camera-space point, then K times it, then the first two rows over
// the third.  (misc.project_pts, used by MSPD, applies K [R|t] to the homogeneous point instead.)
__device__ __forceinline__ void project_rt(const double* M, const double* K, double x, double y, double z, double& u,
                                           double& v) {
  // explicit roundings: the estimate and the GT projections are inlined at two sites, and equal poses must give equal
  // bits (a perfect estimate has error 0, as in the reference)
  double cx, cy, cz;
  xform(M, x, y, z, cx, cy, cz);
  const double a = __fma_rn(K[0], cx, __fma_rn(K[1], cy, __dmul_rn(K[2], cz)));
  const double b = __fma_rn(K[3], cx, __fma_rn(K[4], cy, __dmul_rn(K[5], cz)));
  const double r = __drcp_rn(__fma_rn(K[6], cx, __fma_rn(K[7], cy, __dmul_rn(K[8], cz))));   // a division per row spills
  u = __dmul_rn(a, r);
  v = __dmul_rn(b, r);
}

// grid (P, ceil(max_syms / SYM_BLOCK)): pose_error.arp_2d / arp_2d_sym, the mean over the object's points of the pixel
// distance between the estimate-pose and the GT(-symmetry)-pose projections, min over the symmetries.  Warp w owns
// symmetry w of the block and holds that symmetry's whole sum: lane l adds the distances of points l, l+32, ... in
// order (tiles are a multiple of 32 points), then an xor tree.  So the bits depend on nothing but the pair.
__global__ void __launch_bounds__(SYM_THREADS)
sym_proj_mean_kernel(const double* __restrict__ pts, const int64_t* __restrict__ pt_off, const double* __restrict__ syms,
                     const int64_t* __restrict__ sym_off, const int* __restrict__ pair_obj,
                     const double* __restrict__ pose_est, const double* __restrict__ pose_gt,
                     const double* __restrict__ Ks, const uint8_t* __restrict__ use_syms, double* __restrict__ err) {
  const int p = blockIdx.x, o = pair_obj[p];
  const bool sym = use_syms[p] != 0;
  const int64_t s0 = sym ? sym_off[o] + (int64_t)blockIdx.y * SYM_BLOCK : 0;
  const int ns = sym ? (int)min((int64_t)SYM_BLOCK, sym_off[o + 1] - s0) : (blockIdx.y == 0 ? 1 : 0);
  if (ns <= 0) return;
  __shared__ double s_est[12], s_K[9], s_gs[SYM_BLOCK][12];
  __shared__ double s_tile[5][SYM_THREADS];   // x, y, z, estimate-pose projection u, v
  __shared__ double s_red[SYM_BLOCK];
  if (threadIdx.x < 12) s_est[threadIdx.x] = pose_est[(size_t)p * 12 + threadIdx.x];
  if (threadIdx.x < 9) s_K[threadIdx.x] = Ks[(size_t)p * 9 + threadIdx.x];
  if (threadIdx.x < ns) gt_sym_pose(pose_gt + (size_t)p * 12, sym ? syms + (size_t)(s0 + threadIdx.x) * 12 : nullptr,
                                    s_gs[threadIdx.x]);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ws = min(warp, ns - 1);   // warps past ns idle in the point loop but keep the barriers
  double G[12], K[9];
#pragma unroll
  for (int j = 0; j < 12; ++j) G[j] = s_gs[ws][j];
#pragma unroll
  for (int j = 0; j < 9; ++j) K[j] = s_K[j];
  double sum = 0.0;
  const double* X = pts + (size_t)pt_off[o] * 3;
  const int n = (int)(pt_off[o + 1] - pt_off[o]);
  for (int t0 = 0; t0 < n; t0 += SYM_THREADS) {
    const int cnt = min(SYM_THREADS, n - t0);
    __syncthreads();
    if (threadIdx.x < cnt) {
      const int i = t0 + threadIdx.x;
      const double x = X[i * 3], y = X[i * 3 + 1], z = X[i * 3 + 2];
      double eu, ev;
      project_rt(s_est, K, x, y, z, eu, ev);
      s_tile[0][threadIdx.x] = x; s_tile[1][threadIdx.x] = y; s_tile[2][threadIdx.x] = z;
      s_tile[3][threadIdx.x] = eu; s_tile[4][threadIdx.x] = ev;
    }
    __syncthreads();
    if (warp < ns) {
      for (int j = lane; j < cnt; j += 32) {
        double gu, gv;
        project_rt(G, K, s_tile[0][j], s_tile[1][j], s_tile[2][j], gu, gv);
        const double du = s_tile[3][j] - gu, dv = s_tile[4][j] - gv;
        sum = __dadd_rn(sum, sqrt(du * du + dv * dv));
      }
    }
  }
  sum = warp_sum_d(sum);
  if (lane == 0 && warp < ns) s_red[warp] = sum / (double)n;
  __syncthreads();
  if (threadIdx.x == 0) {
    double best = INFINITY;
    for (int s = 0; s < ns; ++s) best = fmin(best, s_red[s]);
    atomicMin((unsigned long long*)(err + p), (unsigned long long)__double_as_longlong(best));
  }
}

// pose_error.re / re_sym (:359-396): trace(R_e . R_gs^T), clamped to 3, cos = clip(0.5 (trace - 1), -1, 1), in degrees.
__device__ __forceinline__ double rot_err_deg(const double* Pe, const double* G) {
  double tr = 0.0;
  for (int r = 0; r < 3; ++r) tr += Pe[r * 4] * G[r * 4] + Pe[r * 4 + 1] * G[r * 4 + 1] + Pe[r * 4 + 2] * G[r * 4 + 2];
  tr = tr <= 3.0 ? tr : 3.0;
  const double c = fmin(1.0, fmax(-1.0, 0.5 * (tr - 1.0)));
  return acos(c) * (180.0 / M_PI);
}

// One warp per pair, lanes over the symmetry set (or the GT pose alone): pose_error.re(_sym) in degrees and
// te(_sym) = |t_gs - t_e| in the units of t, each minimised over the symmetries on its own (eval_calc_errors.py
// :574-596 calls the two functions separately).
__global__ void __launch_bounds__(RT_THREADS)
sym_rt_kernel(const double* __restrict__ syms, const int64_t* __restrict__ sym_off, const int* __restrict__ pair_obj,
              const double* __restrict__ pose_est, const double* __restrict__ pose_gt,
              const uint8_t* __restrict__ use_syms, int P, double* __restrict__ re_deg, double* __restrict__ te) {
  const int p = blockIdx.x * (RT_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;   // whole warps leave together
  const bool sym = use_syms[p] != 0;
  const int o = pair_obj[p];
  const int64_t s_begin = sym ? sym_off[o] : 0, s_end = sym ? sym_off[o + 1] : 1;
  double Pe[12], Pg[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) { Pe[j] = pose_est[(size_t)p * 12 + j]; Pg[j] = pose_gt[(size_t)p * 12 + j]; }
  double best_r = INFINITY, best_t = INFINITY;
  for (int64_t s = s_begin + lane; s < s_end; s += 32) {
    double G[12];
    gt_sym_pose(Pg, sym ? syms + (size_t)s * 12 : nullptr, G);
    best_r = fmin(best_r, rot_err_deg(Pe, G));
    const double dx = G[3] - Pe[3], dy = G[7] - Pe[7], dz = G[11] - Pe[11];
    best_t = fmin(best_t, sqrt(dx * dx + dy * dy + dz * dz));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    best_r = fmin(best_r, __shfl_xor_sync(0xffffffffu, best_r, off));
    best_t = fmin(best_t, __shfl_xor_sync(0xffffffffu, best_t, off));
  }
  if (lane == 0) { re_deg[p] = best_r; te[p] = best_t; }
}

// Fixed-order CTA sum: xor-tree inside each warp, then the warp sums in warp order.
__device__ __forceinline__ double block_sum_fixed(double v, double* s_red) {
  v = warp_sum_d(v);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < AD_THREADS / 32; ++w) s = __dadd_rn(s, s_red[w]);
  return s;
}

// grid (P, ceil(max_n / AD_THREADS)): the CTA of chunk c sums the distances of points [c*256, c*256+256) of the pair's
// object into partial[p * n_chunks + c].  ADD: |T_e x_i - T_g x_i|.  ADI: min_j |T_g x_i - T_e x_j| (pose_error.adi's
// nearest neighbour of each GT-pose point among the estimate-pose points), found by a brute-force tiled search.
__global__ void __launch_bounds__(AD_THREADS)
ad_partial_kernel(const double* __restrict__ pts, const int64_t* __restrict__ pt_off, const int* __restrict__ pair_obj,
                  const double* __restrict__ pose_est, const double* __restrict__ pose_gt, const uint8_t* __restrict__ use_adi,
                  const uint8_t* __restrict__ gate, int n_chunks, double* __restrict__ partial) {
  const int p = blockIdx.x, c = blockIdx.y, o = pair_obj[p];
  const int n = (int)(pt_off[o + 1] - pt_off[o]);
  if (!gate[p] || c * AD_THREADS >= n) return;
  __shared__ double s_e[12], s_g[12];
  __shared__ double3 s_tile[AD_TILE];
  __shared__ double s_red[AD_THREADS / 32];
  if (threadIdx.x < 12) {
    s_e[threadIdx.x] = pose_est[(size_t)p * 12 + threadIdx.x];
    s_g[threadIdx.x] = pose_gt[(size_t)p * 12 + threadIdx.x];
  }
  __syncthreads();
  const double* X = pts + (size_t)pt_off[o] * 3;
  const int i = c * AD_THREADS + threadIdx.x;
  const bool valid = i < n;
  double gx = 0.0, gy = 0.0, gz = 0.0;
  if (valid) xform(s_g, X[i * 3], X[i * 3 + 1], X[i * 3 + 2], gx, gy, gz);
  double d = 0.0;
  if (!use_adi[p]) {
    if (valid) {
      double ex, ey, ez;
      xform(s_e, X[i * 3], X[i * 3 + 1], X[i * 3 + 2], ex, ey, ez);
      const double dx = ex - gx, dy = ey - gy, dz = ez - gz;
      d = sqrt(dx * dx + dy * dy + dz * dz);
    }
  } else {
    double best = INFINITY;
    for (int j0 = 0; j0 < n; j0 += AD_TILE) {
      const int cnt = min(AD_TILE, n - j0);
      __syncthreads();
      for (int j = threadIdx.x; j < cnt; j += AD_THREADS) {
        double ex, ey, ez;
        xform(s_e, X[(j0 + j) * 3], X[(j0 + j) * 3 + 1], X[(j0 + j) * 3 + 2], ex, ey, ez);
        s_tile[j] = make_double3(ex, ey, ez);
      }
      __syncthreads();
#pragma unroll 4
      for (int j = 0; j < cnt; ++j) {
        const double3 e = s_tile[j];
        const double dx = gx - e.x, dy = gy - e.y, dz = gz - e.z;
        best = fmin(best, dx * dx + dy * dy + dz * dz);
      }
    }
    if (valid) d = sqrt(best);
  }
  const double s = block_sum_fixed(d, s_red);
  if (threadIdx.x == 0) partial[(size_t)p * n_chunks + c] = s;
}

// mean = (sum of the chunk partials in chunk order) / N; gate 0 -> inf (eval_calc_errors.py:426-431)
__global__ void ad_finalize_kernel(const double* __restrict__ partial, const int64_t* __restrict__ pt_off,
                                   const int* __restrict__ pair_obj, const uint8_t* __restrict__ gate, int P, int n_chunks,
                                   double* __restrict__ err) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  if (!gate[p]) {
    err[p] = INFINITY;
    return;
  }
  const int o = pair_obj[p];
  const int n = (int)(pt_off[o + 1] - pt_off[o]);
  double s = 0.0;
  for (int c = 0; c * AD_THREADS < n; ++c) s = __dadd_rn(s, partial[(size_t)p * n_chunks + c]);
  err[p] = s / (double)n;
}

int launch_status() {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gdrn_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
    return GDRN_ERR_CUDA;
  }
  return 0;
}

}  // namespace

extern "C" size_t gdrn_vsd_workspace_bytes(int P, int T) { return (size_t)(P > 0 ? P : 0) * (size_t)(T + 2) * 8; }

extern "C" int gdrn_vsd_errors(const float* depth_est, const float* depth_gt, const float* depth_test, int H, int W,
                               const int* pair_est, const int* pair_gt, const int* pair_img, const double* Ks,
                               const double* diameters, const uint8_t* gate, int P, const double* taus, int T, float delta,
                               int normalized_by_diameter, void* counts_ws, size_t ws_bytes, double* errors, void* stream) {
  GDRN_REQUIRE(depth_est && depth_gt && depth_test && pair_est && pair_gt && pair_img && Ks && diameters && gate && taus &&
                   counts_ws && errors, "vsd: null argument");
  GDRN_REQUIRE(H > 0 && W > 0 && P > 0, "vsd: need H, W, P > 0");
  GDRN_REQUIRE(T >= 1 && T <= VSD_MAX_T, "vsd: need 1 <= T <= 32 taus");
  GDRN_REQUIRE(ws_bytes >= gdrn_vsd_workspace_bytes(P, T), "vsd: counts workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  GDRN_CHECK_CUDA(cudaMemsetAsync(counts_ws, 0, gdrn_vsd_workspace_bytes(P, T), st));
  const long long HW = (long long)H * W;
  const int bx = (int)min((HW + VSD_THREADS * 8 - 1) / (VSD_THREADS * 8), 1024LL);   // ~8 pixels per thread
  vsd_count_kernel<<<dim3(P, bx), VSD_THREADS, 0, st>>>(depth_est, depth_gt, depth_test, H, W, pair_est, pair_gt, pair_img,
                                                        Ks, diameters, gate, taus, T, delta, normalized_by_diameter,
                                                        (unsigned long long*)counts_ws);
  vsd_finalize_kernel<<<(P * T + 255) / 256, 256, 0, st>>>((const unsigned long long*)counts_ws, gate, P, T, errors);
  gdrn_count_launch(2);
  return launch_status();
}

extern "C" int gdrn_sym_max_dist(const double* pts, const int64_t* pt_offsets, const double* syms,
                                 const int64_t* sym_offsets, const int* pair_obj, const double* pose_est,
                                 const double* pose_gt, const double* Ks, const uint8_t* gate_mssd, int P, int max_syms,
                                 double* mssd, double* mspd, void* stream) {
  GDRN_REQUIRE(pts && pt_offsets && syms && sym_offsets && pair_obj && pose_est && pose_gt && Ks && gate_mssd && mssd && mspd,
               "sym_max_dist: null argument");
  GDRN_REQUIRE(P > 0 && max_syms > 0, "sym_max_dist: need P > 0 and max_syms > 0");
  cudaStream_t st = (cudaStream_t)stream;
  sym_init_kernel<<<(P + 255) / 256, 256, 0, st>>>(mssd, mspd, P);
  sym_max_dist_kernel<<<dim3(P, (max_syms + SYM_BLOCK - 1) / SYM_BLOCK), SYM_THREADS, 0, st>>>(
      pts, pt_offsets, syms, sym_offsets, pair_obj, pose_est, pose_gt, Ks, gate_mssd, mssd, mspd);
  gdrn_count_launch(2);
  return launch_status();
}

extern "C" int gdrn_sym_proj_mean(const double* pts, const int64_t* pt_offsets, const double* syms,
                                  const int64_t* sym_offsets, const int* pair_obj, const double* pose_est,
                                  const double* pose_gt, const double* Ks, const uint8_t* use_syms, int P, int max_syms,
                                  double* err, void* stream) {
  GDRN_REQUIRE(pts && pt_offsets && syms && sym_offsets && pair_obj && pose_est && pose_gt && Ks && use_syms && err,
               "sym_proj_mean: null argument");
  GDRN_REQUIRE(P > 0 && max_syms > 0, "sym_proj_mean: need P > 0 and max_syms > 0");
  cudaStream_t st = (cudaStream_t)stream;
  fill_inf_kernel<<<(P + 255) / 256, 256, 0, st>>>(err, P);
  sym_proj_mean_kernel<<<dim3(P, (max_syms + SYM_BLOCK - 1) / SYM_BLOCK), SYM_THREADS, 0, st>>>(
      pts, pt_offsets, syms, sym_offsets, pair_obj, pose_est, pose_gt, Ks, use_syms, err);
  gdrn_count_launch(2);
  return launch_status();
}

extern "C" int gdrn_sym_rt_errors(const double* syms, const int64_t* sym_offsets, const int* pair_obj,
                                  const double* pose_est, const double* pose_gt, const uint8_t* use_syms, int P,
                                  double* re_deg, double* te, void* stream) {
  GDRN_REQUIRE(syms && sym_offsets && pair_obj && pose_est && pose_gt && use_syms && re_deg && te,
               "sym_rt_errors: null argument");
  GDRN_REQUIRE(P > 0, "sym_rt_errors: need P > 0");
  constexpr int pairs_per_cta = RT_THREADS / 32;
  sym_rt_kernel<<<(P + pairs_per_cta - 1) / pairs_per_cta, RT_THREADS, 0, (cudaStream_t)stream>>>(
      syms, sym_offsets, pair_obj, pose_est, pose_gt, use_syms, P, re_deg, te);
  gdrn_count_launch(1);
  return launch_status();
}

extern "C" size_t gdrn_ad_workspace_bytes(int P, int max_pts) {
  if (P <= 0 || max_pts <= 0) return 0;
  return (size_t)P * (size_t)((max_pts + AD_THREADS - 1) / AD_THREADS) * sizeof(double);
}

extern "C" int gdrn_ad_errors(const double* pts, const int64_t* pt_offsets, const int* pair_obj, const double* pose_est,
                              const double* pose_gt, const uint8_t* use_adi, const uint8_t* gate, int P, int max_pts,
                              void* ws, size_t ws_bytes, double* err, void* stream) {
  GDRN_REQUIRE(pts && pt_offsets && pair_obj && pose_est && pose_gt && use_adi && gate && ws && err, "ad: null argument");
  GDRN_REQUIRE(P > 0 && max_pts > 0, "ad: need P > 0 and max_pts > 0");
  GDRN_REQUIRE(ws_bytes >= gdrn_ad_workspace_bytes(P, max_pts), "ad: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int n_chunks = (max_pts + AD_THREADS - 1) / AD_THREADS;
  ad_partial_kernel<<<dim3(P, n_chunks), AD_THREADS, 0, st>>>(pts, pt_offsets, pair_obj, pose_est, pose_gt, use_adi, gate,
                                                             n_chunks, (double*)ws);
  ad_finalize_kernel<<<(P + 255) / 256, 256, 0, st>>>((const double*)ws, pt_offsets, pair_obj, gate, P, n_chunks, err);
  gdrn_count_launch(2);
  return launch_status();
}
