// Batched RANSAC-PnP from dense 2D-3D correspondences (SURVEY.md 8f rank 2): one CTA per ROI.
//
// Replaces the per-ROI host loop of the reference's TEST.USE_PNP path: get_pnp_ransac_pose
// (core/gdrn_modeling/engine/gdrn_evaluator.py:1122-1180: get_out_coor / get_out_mask, correspondence selection
// get_img_model_points_with_coords2d :1183-1221) followed by misc.pnp_v2 (lib/pysixd/misc.py:153-208) =
// cv2.solvePnPRansac(flags=SOLVEPNP_EPNP, reprojectionError=3, iterationsCount=100) -- which GdrnPredictor runs by
// default (core/gdrn_modeling/demo/predictor_gdrn.py:58,169).
//
// Per ROI (all on chip, fp64 geometry):
//   1. L1 mask -> per-ROI min-max normalisation (engine_utils.py:313-333), xyz = (coor - 0.5) * extent, image points =
//      roi_coord_2d * (im_W, im_H); selection mask > thr & |xyz_k| > 1e-4 * extent_k, compacted in row-major order
//      (the order numpy boolean indexing gives the reference).
//   2. `iters` hypotheses: 4 sampled correspondences each (counter-based hash RNG of (seed, roi, hypothesis), or caller
//      supplied indices; four distinct ids, a repeated caller id gives no model), Grunert P3P on the first three (quartic
//      by Ferrari + Newton polish, then Newton on the depths), the fourth picks among the <= 4 solutions; a thread each.
//   3. inlier count of every hypothesis over all correspondences (reprojection error < thr px; a warp per hypothesis,
//      lanes over points), best = max count (lowest index on ties).
//   4. refit on the inliers of the best hypothesis: Levenberg-Marquardt on the reprojection error (6x6 normal equations
//      reduced over the CTA), then the inlier set is recomputed with the refined pose and refitted once more.
// OpenCV's final step is EPnP on the inliers (an algebraic solution + Gauss-Newton); both minimise the same residual, so
// poses agree to the tolerance tests/test_gpu_parity.py states, not bit-exactly.  < 4 correspondences -> the
// reference's sentinel pose (-100 everywhere, gdrn_evaluator.py:1178-1179).
//
// The network-initialised types of TEST.PNP_TYPE (process_net_and_pnp, gdrn_evaluator.py:241-371) reuse steps 1 and 4:
// net_iter_pnp is pnp_iterative_kernel (step 1, then the step-4 LM over all correspondences from the network pose);
// net_ransac_pnp / _rot are pnp_ransac_kernel at 20 iterations followed by pnp_net_select_kernel.
#include "common.cuh"

namespace {

constexpr int PR_THREADS = 512;
constexpr int PR_MAX_PTS = 4096;   // 64 x 64 maps
constexpr int PR_MAX_HYP = 256;
constexpr int PNP_ITERATIVE_MAX_ITERS = 20;   // OpenCV's SOLVEPNP_ITERATIVE cap (cvFindExtrinsicCameraParams2 max_iter)
enum { PNP_NET_ITER = 0, PNP_NET_RANSAC = 1, PNP_NET_RANSAC_ROT = 2 };   // gdrn_pnp_net_maps pnp_type

// Per-stage record of pnp_ransac_kernel (gdrn_pnp_ransac_trace), all device pointers; every member null in production
// calls.  Entries a ROI does not reach (after an early sentinel return) are left as the caller initialised them.
struct PnpTrace {
  int* count;               // [n] selected correspondences N
  int* src;                 // [n, PR_MAX_PTS] source pixel / point of compacted entry i (-1 from N on)
  int* samples;             // [n, iters, 4] ids each hypothesis used (after % N and de-duplication)
  int* nsol;                // [n, iters] P3P solutions
  double* hyp;              // [n, iters, 12] the solution the fourth point chose
  int* cnt;                 // [n, iters] inlier count (-1: no model)
  int* best;                // [n]
  unsigned char* inl;       // [n, 2, PR_MAX_PTS] inlier flags at the start of each refit round, compacted order
  double* round_pose;       // [n, 2, 2, 12] start / end pose of each refit round
  double* round_cost;       // [n, 2, 3] cost at the start, the lowest cost LM evaluated, the cost at the returned pose
  double* pose;             // [n, 12] final pose (-100 for the sentinel)
};

struct PnpParams {
  const float* coor_x; const float* coor_y; const float* coor_z;   // [n, hw*hw] network outputs in [0,1]
  const float* mask;        // [n, hw*hw] raw visible-mask output, or null (then `sel` picks)
  const float* coord2d;     // [n, 2, hw*hw] normalised image coordinates of the ROI grid
  const float* im_hw;       // [n, 2] (im_H, im_W)
  const float* extents;     // [n, 3]
  const float* Ks;          // [n, 9]
  const int* idxs;          // [n, iters, 4] indices into the compacted correspondence list (taken modulo count), or null
  // generic-correspondence entry (pts given directly): pts3d [n, npts, 3], pts2d [n, npts, 2], npts <= PR_MAX_PTS
  const float* pts3d; const float* pts2d;
  int npts;                 // pixels per ROI (hw*hw) or points per problem
  int iters;
  float mask_thr, reproj_thr;
  unsigned seed;
  float* poses;             // [n, 12]
  int* n_inliers;           // [n] (or null)
  unsigned char* inlier_mask;   // [n, npts] over the INPUT pixels/points (or null)
  PnpTrace tr;
};

__device__ __forceinline__ unsigned hash32(unsigned x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// real roots of a4 x^4 + a3 x^3 + a2 x^2 + a1 x + a0 (Ferrari via one positive root of the resolvent cubic), polished
__device__ int solve_quartic(double a4, double a3, double a2, double a1, double a0, double* out) {
  if (fabs(a4) < 1e-300) return 0;
  const double b = a3 / a4, c = a2 / a4, d = a1 / a4, e = a0 / a4;
  const double b2 = b * b;
  const double p = c - 3.0 * b2 / 8.0;
  const double q = d - b * c / 2.0 + b2 * b / 8.0;
  const double r = e - b * d / 4.0 + b2 * c / 16.0 - 3.0 * b2 * b2 / 256.0;
  double y[4];
  int n = 0;
  if (fabs(q) < 1e-14 * fmax(1.0, pow(fabs(p), 1.5))) {
    const double disc = p * p - 4.0 * r;
    if (disc >= 0.0) {
      const double s = sqrt(disc);
      const double z0 = (-p + s) / 2.0, z1 = (-p - s) / 2.0;
      if (z0 >= 0.0) { y[n++] = sqrt(z0); y[n++] = -sqrt(z0); }
      if (z1 >= 0.0) { y[n++] = sqrt(z1); y[n++] = -sqrt(z1); }
    }
  } else {
    const double A = p, B = p * p / 4.0 - r, C = -q * q / 8.0;
    const double P = B - A * A / 3.0, Q = 2.0 * A * A * A / 27.0 - A * B / 3.0 + C;
    const double D = Q * Q / 4.0 + P * P * P / 27.0;
    double m;
    if (D >= 0.0) {
      const double sD = sqrt(D);
      m = cbrt(-Q / 2.0 + sD) + cbrt(-Q / 2.0 - sD) - A / 3.0;
    } else {
      const double rho = sqrt(-P * P * P / 27.0);
      const double th = acos(fmax(-1.0, fmin(1.0, -Q / (2.0 * rho))));
      const double mm = 2.0 * sqrt(-P / 3.0);
      m = -1e300;
      for (int k = 0; k < 3; ++k) m = fmax(m, mm * cos((th + 6.283185307179586 * k) / 3.0) - A / 3.0);
    }
    for (int it = 0; it < 2; ++it) {
      const double fm = ((m + A) * m + B) * m + C, dfm = (3.0 * m + 2.0 * A) * m + B;
      if (dfm != 0.0) m -= fm / dfm;
    }
    if (m <= 0.0) return 0;
    const double s = sqrt(2.0 * m);
    for (int sg = 1; sg >= -1; sg -= 2) {
      const double cc = p / 2.0 + m - sg * q / (2.0 * s);
      const double disc = s * s - 4.0 * cc;
      // a double root rounded into a complex pair is still a root: keep it within a relative 1e-9 (p3p_grunert's
      // depth refinement then settles it or drops it)
      if (disc >= -1e-9 * (s * s + fabs(4.0 * cc))) {
        const double sd = sqrt(fmax(disc, 0.0));
        y[n++] = (-sg * s + sd) / 2.0;
        y[n++] = (-sg * s - sd) / 2.0;
      }
    }
  }
  for (int i = 0; i < n; ++i) {
    double x = y[i] - b / 4.0;
    for (int it = 0; it < 2; ++it) {
      const double fx = (((a4 * x + a3) * x + a2) * x + a1) * x + a0;
      const double dfx = ((4.0 * a4 * x + 3.0 * a3) * x + 2.0 * a2) * x + a1;
      if (dfx != 0.0) x -= fx / dfx;
    }
    out[i] = x;
  }
  return n;
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double norm3(const double* a) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }

// orthonormal frame (columns e1, e2, e3) of the triangle X0 X1 X2; false if degenerate
__device__ bool tri_frame(const double* X0, const double* X1, const double* X2, double* F /*[9] row-major, columns = e*/) {
  double e1[3] = {X1[0] - X0[0], X1[1] - X0[1], X1[2] - X0[2]};
  double n1 = norm3(e1);
  if (n1 < 1e-12) return false;
  e1[0] /= n1; e1[1] /= n1; e1[2] /= n1;
  double w[3] = {X2[0] - X0[0], X2[1] - X0[1], X2[2] - X0[2]};
  double e3[3];
  cross3(e1, w, e3);
  double n3 = norm3(e3);
  if (n3 < 1e-12) return false;
  e3[0] /= n3; e3[1] /= n3; e3[2] /= n3;
  double e2[3];
  cross3(e3, e1, e2);
  for (int i = 0; i < 3; ++i) { F[i * 3] = e1[i]; F[i * 3 + 1] = e2[i]; F[i * 3 + 2] = e3[i]; }
  return true;
}

// Grunert P3P: world points P[3][3], unit bearings f[3][3] -> up to 4 (R, t) with x_cam = R X + t; returns count
__device__ int p3p_grunert(const double (*P)[3], const double (*f)[3], double (*Rt)[12]) {
  double d12[3] = {P[1][0] - P[2][0], P[1][1] - P[2][1], P[1][2] - P[2][2]};
  double d02[3] = {P[0][0] - P[2][0], P[0][1] - P[2][1], P[0][2] - P[2][2]};
  double d01[3] = {P[0][0] - P[1][0], P[0][1] - P[1][1], P[0][2] - P[1][2]};
  const double a2 = d12[0] * d12[0] + d12[1] * d12[1] + d12[2] * d12[2];
  const double b2 = d02[0] * d02[0] + d02[1] * d02[1] + d02[2] * d02[2];
  const double c2 = d01[0] * d01[0] + d01[1] * d01[1] + d01[2] * d01[2];
  if (a2 < 1e-18 || b2 < 1e-18 || c2 < 1e-18) return 0;
  const double ca = f[1][0] * f[2][0] + f[1][1] * f[2][1] + f[1][2] * f[2][2];
  const double cb = f[0][0] * f[2][0] + f[0][1] * f[2][1] + f[0][2] * f[2][2];
  const double cg = f[0][0] * f[1][0] + f[0][1] * f[1][1] + f[0][2] * f[1][2];
  const double q = (a2 - c2) / b2, r = (a2 + c2) / b2;
  const double A4 = (q - 1.0) * (q - 1.0) - 4.0 * c2 / b2 * ca * ca;
  const double A3 = 4.0 * (q * (1.0 - q) * cb - (1.0 - r) * ca * cg + 2.0 * c2 / b2 * ca * ca * cb);
  const double A2 = 2.0 * (q * q - 1.0 + 2.0 * q * q * cb * cb + 2.0 * (b2 - c2) / b2 * ca * ca - 4.0 * r * ca * cb * cg +
                           2.0 * (b2 - a2) / b2 * cg * cg);
  const double A1 = 4.0 * (-q * (1.0 + q) * cb + 2.0 * a2 / b2 * cg * cg * cb - (1.0 - r) * ca * cg);
  const double A0 = (1.0 + q) * (1.0 + q) - 4.0 * a2 / b2 * cg * cg;
  double roots[4];
  const int nr = solve_quartic(A4, A3, A2, A1, A0, roots);
  double Fw[9];
  if (!tri_frame(P[0], P[1], P[2], Fw)) return 0;
  int ns = 0;
  for (int i = 0; i < nr; ++i) {
    const double v = roots[i];
    if (!(v > 0.0)) continue;
    const double den = 2.0 * (cg - v * ca);
    if (fabs(den) < 1e-12) continue;
    const double u = ((-1.0 + q) * v * v - 2.0 * q * cb * v + 1.0 + q) / den;
    if (!(u > 0.0)) continue;
    const double s1sq = c2 / (1.0 + u * u - 2.0 * u * cg);
    if (!(s1sq > 0.0)) continue;
    double s1 = sqrt(s1sq), s2 = u * s1, s3 = v * s1;
    // Grunert's quartic loses precision when the bearings are close (samples a few pixels apart): Newton on the three
    // depths with the law-of-cosines system s_i^2 + s_j^2 - 2 cos_ij s_i s_j = d_ij^2 restores it.
    for (int it = 0; it < 3; ++it) {
      const double F0 = s1 * s1 + s2 * s2 - 2.0 * cg * s1 * s2 - c2;   // pair (0, 1)
      const double F1 = s1 * s1 + s3 * s3 - 2.0 * cb * s1 * s3 - b2;   // pair (0, 2)
      const double F2 = s2 * s2 + s3 * s3 - 2.0 * ca * s2 * s3 - a2;   // pair (1, 2)
      const double j00 = 2.0 * (s1 - cg * s2), j01 = 2.0 * (s2 - cg * s1);
      const double j10 = 2.0 * (s1 - cb * s3), j12 = 2.0 * (s3 - cb * s1);
      const double j21 = 2.0 * (s2 - ca * s3), j22 = 2.0 * (s3 - ca * s2);
      // J = [[j00, j01, 0], [j10, 0, j12], [0, j21, j22]]: Cramer's rule
      const double det = j00 * (-j12 * j21) - j01 * (j10 * j22);
      if (!(fabs(det) > 1e-300)) break;
      const double d1 = (F0 * (-j12 * j21) - j01 * (F1 * j22 - j12 * F2)) / det;
      const double d2 = (j00 * (F1 * j22 - j12 * F2) - F0 * (j10 * j22)) / det;
      const double d3 = (F0 * (j10 * j21) - j00 * (j21 * F1) - j01 * (j10 * F2)) / det;
      s1 -= d1; s2 -= d2; s3 -= d3;
    }
    {   // a candidate the refinement did not bring onto the system is not a pose
      const double r0 = s1 * s1 + s2 * s2 - 2.0 * cg * s1 * s2 - c2, r1 = s1 * s1 + s3 * s3 - 2.0 * cb * s1 * s3 - b2;
      const double r2 = s2 * s2 + s3 * s3 - 2.0 * ca * s2 * s3 - a2;
      if (!(s1 > 0.0 && s2 > 0.0 && s3 > 0.0 && fabs(r0) <= 1e-6 * c2 && fabs(r1) <= 1e-6 * b2 && fabs(r2) <= 1e-6 * a2)) continue;
    }
    double Q0[3] = {s1 * f[0][0], s1 * f[0][1], s1 * f[0][2]};
    double Q1[3] = {s2 * f[1][0], s2 * f[1][1], s2 * f[1][2]};
    double Q2[3] = {s3 * f[2][0], s3 * f[2][1], s3 * f[2][2]};
    double Fc[9];
    if (!tri_frame(Q0, Q1, Q2, Fc)) continue;
    double* o = Rt[ns];
    for (int rr = 0; rr < 3; ++rr)
      for (int cc = 0; cc < 3; ++cc)
        o[rr * 4 + cc] = Fc[rr * 3] * Fw[cc * 3] + Fc[rr * 3 + 1] * Fw[cc * 3 + 1] + Fc[rr * 3 + 2] * Fw[cc * 3 + 2];
    for (int rr = 0; rr < 3; ++rr)
      o[rr * 4 + 3] = (rr == 0 ? Q0[0] : rr == 1 ? Q0[1] : Q0[2]) - (o[rr * 4] * P[0][0] + o[rr * 4 + 1] * P[0][1] + o[rr * 4 + 2] * P[0][2]);
    ++ns;
  }
  return ns;
}

__device__ __forceinline__ bool project(const double* Rt, const double* K, float X, float Y, float Z, double* u, double* v) {
  const double xc = Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Rt[3];
  const double yc = Rt[4] * X + Rt[5] * Y + Rt[6] * Z + Rt[7];
  const double zc = Rt[8] * X + Rt[9] * Y + Rt[10] * Z + Rt[11];
  if (!(zc > 1e-9)) return false;
  *u = K[0] * xc / zc + K[1] * yc / zc + K[2];
  *v = K[4] * yc / zc + K[5];
  return true;
}

// symmetric 6x6 solve (A + lambda diag(A)) x = g by Cholesky; false if not positive definite
__device__ bool solve6(const double* A, const double* g, double lambda, double* x) {
  double L[36];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = A[i * 6 + j];
      if (i == j) s += lambda * fmax(A[i * 6 + i], 1e-12);
      for (int k = 0; k < j; ++k) s -= L[i * 6 + k] * L[j * 6 + k];
      if (i == j) {
        if (!(s > 0.0)) return false;
        L[i * 6 + i] = sqrt(s);
      } else {
        L[i * 6 + j] = s / L[j * 6 + j];
      }
    }
  double yv[6];
  for (int i = 0; i < 6; ++i) {
    double s = g[i];
    for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * yv[k];
    yv[i] = s / L[i * 6 + i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = yv[i];
    for (int k = i + 1; k < 6; ++k) s -= L[k * 6 + i] * x[k];
    x[i] = s / L[i * 6 + i];
  }
  return true;
}

// R <- exp([w]x) R  (Rodrigues), t <- t + dt
__device__ void apply_update(double* Rt, const double* d) {
  const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  double E[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (th > 1e-14) {
    const double kx = d[0] / th, ky = d[1] / th, kz = d[2] / th, c = cos(th), s = sin(th), C = 1.0 - c;
    E[0] = c + kx * kx * C; E[1] = kx * ky * C - kz * s; E[2] = kx * kz * C + ky * s;
    E[3] = ky * kx * C + kz * s; E[4] = c + ky * ky * C; E[5] = ky * kz * C - kx * s;
    E[6] = kz * kx * C - ky * s; E[7] = kz * ky * C + kx * s; E[8] = c + kz * kz * C;
  }
  double Rn[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Rn[r * 3 + c] = E[r * 3] * Rt[c] + E[r * 3 + 1] * Rt[4 + c] + E[r * 3 + 2] * Rt[8 + c];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) Rt[r * 4 + c] = Rn[r * 3 + c];
    Rt[r * 4 + 3] += d[3 + r];
  }
}

// Shared-memory workspace of one ROI's correspondences (the dynamic smem of both PnP kernels) and of the CTA reductions.
struct PnpShared {
  float* s3;                      // [PR_MAX_PTS][3] model points
  float* s2;                      // [PR_MAX_PTS][2] image points
  unsigned short* s_src;          // [PR_MAX_PTS] source pixel / point of entry i
  double (*s_red)[28];            // [PR_THREADS / 32][28] per-warp partial sums
  double* s_K;                    // [9]
  double* s_step;                 // [8] LM decisions broadcast by thread 0
  float* s_mm;                    // [2] mask min / max
  int* s_count;
  int* s_scan;                    // [PR_THREADS / 32 + 1]
};

// Step 1 of both kernels: the selected correspondences of ROI `roi` compacted into sh.s3 / s2 / s_src in row-major
// order; returns their count (in every thread).
__device__ __forceinline__ int gather_correspondences(const PnpParams& p, int roi, const PnpShared& sh) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int npts = p.npts;
  float* s3 = sh.s3;
  float* s2 = sh.s2;
  unsigned short* s_src = sh.s_src;
  double (*s_red)[28] = sh.s_red;
  float* s_mm = sh.s_mm;
  int& s_count = *sh.s_count;
  int* s_scan = sh.s_scan;
  if (p.pts3d == nullptr) {
    float mn = INFINITY, mx = -INFINITY;
    for (int i = tid; i < npts; i += PR_THREADS) {
      const float m = p.mask[(long long)roi * npts + i];
      mn = fminf(mn, m); mx = fmaxf(mx, m);
    }
    for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if (lane == 0) { reinterpret_cast<float*>(s_red)[warp * 2] = mn; reinterpret_cast<float*>(s_red)[warp * 2 + 1] = mx; }
    __syncthreads();
    if (tid == 0) {
      float a = INFINITY, b = -INFINITY;
      for (int w = 0; w < PR_THREADS / 32; ++w) { a = fminf(a, reinterpret_cast<float*>(s_red)[w * 2]); b = fmaxf(b, reinterpret_cast<float*>(s_red)[w * 2 + 1]); }
      s_mm[0] = a; s_mm[1] = b;
    }
    __syncthreads();
  }
  {
    // ordered compaction: chunks of PR_THREADS pixels, block-wide exclusive scan of the selection flags
    const float ex = p.extents ? p.extents[roi * 3] : 0.f, ey = p.extents ? p.extents[roi * 3 + 1] : 0.f, ez = p.extents ? p.extents[roi * 3 + 2] : 0.f;
    const float imH = p.im_hw ? p.im_hw[roi * 2] : 1.f, imW = p.im_hw ? p.im_hw[roi * 2 + 1] : 1.f;
    if (tid == 0) s_count = 0;
    __syncthreads();
    for (int base = 0; base < npts; base += PR_THREADS) {
      const int i = base + tid;
      bool sel = false;
      float X = 0.f, Y = 0.f, Z = 0.f, U = 0.f, V = 0.f;
      if (i < npts) {
        if (p.pts3d) {
          X = p.pts3d[((long long)roi * npts + i) * 3]; Y = p.pts3d[((long long)roi * npts + i) * 3 + 1]; Z = p.pts3d[((long long)roi * npts + i) * 3 + 2];
          U = p.pts2d[((long long)roi * npts + i) * 2]; V = p.pts2d[((long long)roi * npts + i) * 2 + 1];
          sel = true;
        } else {
          // get_out_mask (L1): (m - min) / (max - min); xyz denormalisation and image points: gdrn_evaluator.py:1196-1212
          const float m = (p.mask[(long long)roi * npts + i] - s_mm[0]) / (s_mm[1] - s_mm[0]);
          X = (p.coor_x[(long long)roi * npts + i] - 0.5f) * ex;
          Y = (p.coor_y[(long long)roi * npts + i] - 0.5f) * ey;
          Z = (p.coor_z[(long long)roi * npts + i] - 0.5f) * ez;
          U = p.coord2d[((long long)roi * 2) * npts + i] * imW;
          V = p.coord2d[((long long)roi * 2 + 1) * npts + i] * imH;
          sel = (m > p.mask_thr) && (fabsf(X) > 0.0001f * ex) && (fabsf(Y) > 0.0001f * ey) && (fabsf(Z) > 0.0001f * ez);
        }
      }
      const unsigned bal = __ballot_sync(0xffffffffu, sel);
      if (lane == 0) s_scan[warp] = __popc(bal);
      __syncthreads();
      if (tid == 0) {
        int acc = s_count;
        for (int w = 0; w < PR_THREADS / 32; ++w) { const int c = s_scan[w]; s_scan[w] = acc; acc += c; }
        s_scan[PR_THREADS / 32] = acc;
      }
      __syncthreads();
      if (sel) {
        const int slot = s_scan[warp] + __popc(bal & ((1u << lane) - 1u));
        s3[slot * 3] = X; s3[slot * 3 + 1] = Y; s3[slot * 3 + 2] = Z;
        s2[slot * 2] = U; s2[slot * 2 + 1] = V;
        s_src[slot] = (unsigned short)i;
      }
      __syncthreads();
      if (tid == 0) s_count = s_scan[PR_THREADS / 32];
      __syncthreads();
    }
  }
  return s_count;
}

// Levenberg-Marquardt on the reprojection error of the N compacted correspondences (those with inl[i] != 0, or all of
// them when inl is null), starting from and updating s_pose [12] in place; s_save [12] holds the last accepted pose.
// Every thread must call it; thread 0 makes the decisions.
//   kFromGuess = false (RANSAC refit): points at z <= 1e-9 are left out, at most `max_iters` normal-equation solves.
//   kFromGuess = true (network-initialised PnP): like OpenCV's iterative solver, every point with z != 0 counts (from a
//     poor start some may lie behind the camera; dropping them would reward steps that push points there), and only
//     accepted steps count towards `max_iters` (at most 4 * max_iters solves in all).
// The cost lm_refine minimises (sum of squared reprojection errors over the same points) at s_pose, summed in the order
// lm_refine sums it; returned in every thread.  Every thread must call it.
template <bool kFromGuess>
__device__ double pose_cost(const double* s_pose, const unsigned char* inl, int N, const PnpShared& sh) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* s3 = sh.s3;
  const float* s2 = sh.s2;
  const double* s_K = sh.s_K;
  double acc = 0.0;
  for (int i = tid; i < N; i += PR_THREADS) {
    if (inl && !inl[i]) continue;
    const double X = s3[i * 3], Y = s3[i * 3 + 1], Z = s3[i * 3 + 2];
    const double xc = s_pose[0] * X + s_pose[1] * Y + s_pose[2] * Z + s_pose[3];
    const double yc = s_pose[4] * X + s_pose[5] * Y + s_pose[6] * Z + s_pose[7];
    const double zc = s_pose[8] * X + s_pose[9] * Y + s_pose[10] * Z + s_pose[11];
    if (kFromGuess ? zc == 0.0 : !(zc > 1e-9)) continue;
    const double iz = 1.0 / zc;
    const double eu = s_K[0] * xc * iz + s_K[1] * yc * iz + s_K[2] - s2[i * 2], ev = s_K[4] * yc * iz + s_K[5] - s2[i * 2 + 1];
    acc += eu * eu + ev * ev;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __syncthreads();   // s_red may still be read by the caller's last reduction
  if (lane == 0) sh.s_red[warp][0] = acc;
  __syncthreads();
  double tot = 0.0;
  for (int w = 0; w < PR_THREADS / 32; ++w) tot += sh.s_red[w][0];
  __syncthreads();
  return tot;
}

// trace_cost (global [3], or null): cost at the start, the lowest cost evaluated, the cost at the returned pose.
template <bool kFromGuess>
__device__ __forceinline__ void lm_refine(double* s_pose, double* s_save, const unsigned char* inl, int N, int max_iters,
                                          const PnpShared& sh, double* trace_cost = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* s3 = sh.s3;
  const float* s2 = sh.s2;
  const double* s_K = sh.s_K;
  double (*s_red)[28] = sh.s_red;
  double* s_step = sh.s_step;
  double lambda = 1e-4, prev_cost = -1.0, lowest = INFINITY;   // lowest: thread 0's least cost evaluated
  bool pending = false;   // the pose holds a step whose cost has not been evaluated
  for (int it = 0, solves = 0; it < max_iters && solves < 4 * max_iters; ++it, ++solves) {
    // normal equations: 21 (upper JtJ) + 6 (Jt r) + 1 (cost) sums
    double acc[28];
    for (int k = 0; k < 28; ++k) acc[k] = 0.0;
    for (int i = tid; i < N; i += PR_THREADS) {
      if (inl && !inl[i]) continue;
      const double X = s3[i * 3], Y = s3[i * 3 + 1], Z = s3[i * 3 + 2];
      const double rx = s_pose[0] * X + s_pose[1] * Y + s_pose[2] * Z;
      const double ry = s_pose[4] * X + s_pose[5] * Y + s_pose[6] * Z;
      const double rz = s_pose[8] * X + s_pose[9] * Y + s_pose[10] * Z;
      const double xc = rx + s_pose[3], yc = ry + s_pose[7], zc = rz + s_pose[11];
      if (kFromGuess ? zc == 0.0 : !(zc > 1e-9)) continue;
      const double iz = 1.0 / zc;
      const double u = s_K[0] * xc * iz + s_K[1] * yc * iz + s_K[2], v = s_K[4] * yc * iz + s_K[5];
      const double eu = u - s2[i * 2], ev = v - s2[i * 2 + 1];
      // d(u,v)/d(xc,yc,zc)
      const double ux = s_K[0] * iz, uy = s_K[1] * iz, uz = -(s_K[0] * xc + s_K[1] * yc) * iz * iz;
      const double vy = s_K[4] * iz, vz = -s_K[4] * yc * iz * iz;
      // d xc / d w = -[R X]x  (left perturbation), d xc / d t = I
      double Ju[6], Jv[6];
      Ju[0] = uy * (-rz) + uz * ry;           // column 0 of -[r]x = (0, -rz... ) see below
      Ju[1] = ux * rz + uz * (-rx);
      Ju[2] = ux * (-ry) + uy * rx;
      Jv[0] = vy * (-rz) + vz * ry;
      Jv[1] = vz * (-rx);
      Jv[2] = vy * rx;
      Ju[3] = ux; Ju[4] = uy; Ju[5] = uz;
      Jv[3] = 0.0; Jv[4] = vy; Jv[5] = vz;
      int k = 0;
      for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) acc[k++] += Ju[a] * Ju[b] + Jv[a] * Jv[b];
      for (int a = 0; a < 6; ++a) acc[21 + a] += Ju[a] * eu + Jv[a] * ev;
      acc[27] += eu * eu + ev * ev;
    }
    for (int k = 0; k < 28; ++k)
      for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
    if (lane == 0) for (int k = 0; k < 28; ++k) s_red[warp][k] = acc[k];
    __syncthreads();
    if (tid == 0) {
      double tot[28];
      for (int k = 0; k < 28; ++k) { tot[k] = 0.0; for (int w = 0; w < PR_THREADS / 32; ++w) tot[k] += s_red[w][k]; }
      double A[36], g[6], dx[6];
      int k = 0;
      for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) { A[a * 6 + b] = tot[k]; A[b * 6 + a] = tot[k]; ++k; }
      for (int a = 0; a < 6; ++a) g[a] = -tot[21 + a];
      const double cost = tot[27];
      if (trace_cost && prev_cost < 0.0) trace_cost[0] = cost;
      lowest = fmin(lowest, cost);
      int stop = 0;
      if (prev_cost >= 0.0 && cost > prev_cost) {
        // the previous step made it worse: undo it and raise the damping
        for (int a = 0; a < 12; ++a) s_pose[a] = s_save[a];
        lambda *= 10.0;
        s_step[6] = 0.0;   // do not update prev_cost
        stop = lambda > 1e6;
        s_step[7] = stop ? 1.0 : 2.0;   // 2 = retry with the saved pose (normal equations recomputed next iteration)
      } else {
        for (int a = 0; a < 12; ++a) s_save[a] = s_pose[a];   // save
        if (solve6(A, g, lambda, dx)) {
          apply_update(s_pose, dx);
          double nrm = 0.0;
          for (int a = 0; a < 6; ++a) nrm += dx[a] * dx[a];
          stop = nrm < 1e-20;
          lambda = fmax(lambda * 0.3, 1e-9);
        } else {
          lambda *= 10.0;
          stop = lambda > 1e6;
        }
        s_step[6] = 1.0;
        s_step[5] = cost;
        s_step[7] = stop ? 1.0 : 0.0;
      }
    }
    __syncthreads();
    const bool accepted = s_step[6] != 0.0;
    if (accepted) prev_cost = s_step[5];
    pending = accepted;
    const bool stop = s_step[7] == 1.0;
    __syncthreads();
    if (stop) break;
    if (kFromGuess && !accepted) --it;   // a rejected step does not count
  }
  if (pending) {   // the loop ended on a step it never evaluated: keep it only if it did not raise the cost
    const double c = pose_cost<kFromGuess>(s_pose, inl, N, sh);
    if (tid == 0) {
      lowest = fmin(lowest, c);
      if (c > prev_cost) for (int a = 0; a < 12; ++a) s_pose[a] = s_save[a];
    }
    __syncthreads();
  }
  if (trace_cost) {
    const double c = pose_cost<kFromGuess>(s_pose, inl, N, sh);
    if (tid == 0) { trace_cost[1] = lowest; trace_cost[2] = c; }
  }
}

__global__ void __launch_bounds__(PR_THREADS)
pnp_ransac_kernel(const PnpParams p) {
  extern __shared__ float sm_f[];
  float* s3 = sm_f;                         // [PR_MAX_PTS][3] model points
  float* s2 = s3 + 3 * PR_MAX_PTS;          // [PR_MAX_PTS][2] image points
  unsigned short* s_src = reinterpret_cast<unsigned short*>(s2 + 2 * PR_MAX_PTS);   // [PR_MAX_PTS] source pixel of entry i
  unsigned char* s_inl = reinterpret_cast<unsigned char*>(s_src + PR_MAX_PTS);      // [PR_MAX_PTS] inlier flags
  __shared__ double s_hyp[PR_MAX_HYP][12];
  __shared__ int s_cnt[PR_MAX_HYP];
  __shared__ double s_red[PR_THREADS / 32][28];
  __shared__ double s_pose[12], s_K[9], s_step[8];
  __shared__ float s_mm[2];
  __shared__ int s_count, s_scan[PR_THREADS / 32 + 1], s_flag;
  const PnpShared sh = {s3, s2, s_src, s_red, s_K, s_step, s_mm, &s_count, s_scan};

  const int roi = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int npts = p.npts;
  if (tid < 9) s_K[tid] = (double)p.Ks[roi * 9 + tid];

  // ---------------- 1. correspondences ----------------
  const int N = gather_correspondences(p, roi, sh);
  float* out = p.poses + (long long)roi * 12;
  const PnpTrace& tr = p.tr;
  const bool trace = tr.count != nullptr;
  if (trace) {
    if (tid == 0) tr.count[roi] = N;
    for (int i = tid; i < PR_MAX_PTS; i += PR_THREADS) tr.src[(long long)roi * PR_MAX_PTS + i] = i < N ? (int)s_src[i] : -1;
  }
  if (p.inlier_mask) for (int i = tid; i < npts; i += PR_THREADS) p.inlier_mask[(long long)roi * npts + i] = 0;
  if (N < 4) {   // gdrn_evaluator.py:1178-1179
    if (tid < 12) out[tid] = -100.f;
    if (trace && tid < 12) tr.pose[roi * 12 + tid] = -100.0;
    if (tid == 0 && p.n_inliers) p.n_inliers[roi] = 0;
    return;
  }

  // ---------------- 2. hypotheses: one thread each ----------------
  const int H = p.iters;
  const double ifx = 1.0 / s_K[0], ify = 1.0 / s_K[4];
  for (int h = tid; h < H; h += PR_THREADS) {
    int id[4];
    bool distinct = true;
    if (p.idxs) {
      for (int k = 0; k < 4; ++k) id[k] = (int)((unsigned)p.idxs[((long long)roi * H + h) * 4 + k] % (unsigned)N);
      for (int k = 1; k < 4; ++k)
        for (int j = 0; j < k; ++j) distinct = distinct && id[j] != id[k];
    } else {
      unsigned st = hash32(p.seed ^ hash32((unsigned)roi * 0x9E3779B9u + (unsigned)h));
      for (int k = 0; k < 4; ++k) {
        bool dup = true;
        for (int tries = 0; tries < 8 && dup; ++tries) {
          st = hash32(st + 0x6D2B79F5u);
          id[k] = (int)(st % (unsigned)N);
          dup = false;
          for (int j = 0; j < k; ++j) dup = dup || (id[j] == id[k]);
        }
        while (dup) {   // eight draws collided: the next free id (N >= 4, so one exists) keeps the four distinct
          id[k] = id[k] + 1 == N ? 0 : id[k] + 1;
          dup = false;
          for (int j = 0; j < k; ++j) dup = dup || (id[j] == id[k]);
        }
      }
    }
    double P[3][3], f[3][3];
    for (int k = 0; k < 3; ++k) {
      P[k][0] = s3[id[k] * 3]; P[k][1] = s3[id[k] * 3 + 1]; P[k][2] = s3[id[k] * 3 + 2];
      const double yn = ((double)s2[id[k] * 2 + 1] - s_K[5]) * ify;
      const double xn = ((double)s2[id[k] * 2] - s_K[2] - s_K[1] * yn) * ifx;
      const double nn = sqrt(xn * xn + yn * yn + 1.0);
      f[k][0] = xn / nn; f[k][1] = yn / nn; f[k][2] = 1.0 / nn;
    }
    double sols[4][12];
    const int ns = distinct ? p3p_grunert(P, f, sols) : 0;   // a repeated correspondence gives no model
    double best = 1e300;
    int bi = -1;
    for (int s = 0; s < ns; ++s) {
      double u, v;
      if (!project(sols[s], s_K, s3[id[3] * 3], s3[id[3] * 3 + 1], s3[id[3] * 3 + 2], &u, &v)) continue;
      const double du = u - s2[id[3] * 2], dv = v - s2[id[3] * 2 + 1];
      const double e = du * du + dv * dv;
      if (e < best) { best = e; bi = s; }
    }
    if (bi >= 0) {
      for (int k = 0; k < 12; ++k) s_hyp[h][k] = sols[bi][k];
      s_cnt[h] = 0;
    } else {
      s_cnt[h] = -1;   // no valid model from this sample
    }
    if (trace) {
      const long long rh = (long long)roi * H + h;
      for (int k = 0; k < 4; ++k) tr.samples[rh * 4 + k] = id[k];
      tr.nsol[rh] = ns;
      if (bi >= 0) for (int k = 0; k < 12; ++k) tr.hyp[rh * 12 + k] = sols[bi][k];
    }
  }
  __syncthreads();

  // ---------------- 3. inlier counts: a warp per hypothesis ----------------
  const double thr2 = (double)p.reproj_thr * (double)p.reproj_thr;
  for (int h = warp; h < H; h += PR_THREADS / 32) {
    if (s_cnt[h] < 0) continue;
    int c = 0;
    for (int i = lane; i < N; i += 32) {
      double u, v;
      if (project(s_hyp[h], s_K, s3[i * 3], s3[i * 3 + 1], s3[i * 3 + 2], &u, &v)) {
        const double du = u - s2[i * 2], dv = v - s2[i * 2 + 1];
        c += (du * du + dv * dv < thr2) ? 1 : 0;
      }
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_cnt[h] = c;
  }
  __syncthreads();
  if (tid == 0) {
    int bh = -1, bc = -1;
    for (int h = 0; h < H; ++h)
      if (s_cnt[h] > bc) { bc = s_cnt[h]; bh = h; }
    s_flag = bh;
    if (bh >= 0) for (int k = 0; k < 12; ++k) s_pose[k] = s_hyp[bh][k];
    if (trace) tr.best[roi] = bh;
  }
  __syncthreads();
  if (trace) for (int h = tid; h < H; h += PR_THREADS) tr.cnt[(long long)roi * H + h] = s_cnt[h];
  if (s_flag < 0 || s_cnt[s_flag] < 4) {   // RANSAC found no model: the reference's solvePnPRansac returns garbage/false here
    if (tid < 12) out[tid] = -100.f;
    if (trace && tid < 12) tr.pose[roi * 12 + tid] = -100.0;
    if (tid == 0 && p.n_inliers) p.n_inliers[roi] = 0;
    return;
  }

  // ---------------- 4. refit on the inliers (LM), twice ----------------
  for (int round = 0; round < 2; ++round) {
    for (int i = tid; i < N; i += PR_THREADS) {
      double u, v;
      bool in = false;
      if (project(s_pose, s_K, s3[i * 3], s3[i * 3 + 1], s3[i * 3 + 2], &u, &v)) {
        const double du = u - s2[i * 2], dv = v - s2[i * 2 + 1];
        in = du * du + dv * dv < thr2;
      }
      s_inl[i] = in ? 1 : 0;
      if (trace) tr.inl[((long long)roi * 2 + round) * PR_MAX_PTS + i] = in ? 1 : 0;
    }
    __syncthreads();
    double* rp = trace ? tr.round_pose + ((long long)roi * 2 + round) * 24 : nullptr;
    if (trace && tid < 12) rp[tid] = s_pose[tid];
    // s_hyp[0] doubles as the saved pose
    lm_refine<false>(s_pose, s_hyp[0], s_inl, N, 12, sh, trace ? tr.round_cost + ((long long)roi * 2 + round) * 3 : nullptr);
    __syncthreads();
    if (trace && tid < 12) rp[12 + tid] = s_pose[tid];
  }
  // final inlier set of the refined pose
  int cnt = 0;
  for (int i = tid; i < N; i += PR_THREADS) {
    double u, v;
    bool in = false;
    if (project(s_pose, s_K, s3[i * 3], s3[i * 3 + 1], s3[i * 3 + 2], &u, &v)) {
      const double du = u - s2[i * 2], dv = v - s2[i * 2 + 1];
      in = du * du + dv * dv < thr2;
    }
    cnt += in ? 1 : 0;
    if (in && p.inlier_mask) p.inlier_mask[(long long)roi * npts + s_src[i]] = 1;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) s_scan[warp] = cnt;
  __syncthreads();
  if (tid == 0) {
    int c = 0;
    for (int w = 0; w < PR_THREADS / 32; ++w) c += s_scan[w];
    if (p.n_inliers) p.n_inliers[roi] = c;
  }
  if (tid < 12) out[tid] = (float)s_pose[tid];
  if (trace && tid < 12) tr.pose[roi * 12 + tid] = s_pose[tid];
}

// Network-initialised iterative PnP (TEST.PNP_TYPE = "net_iter_pnp", gdrn_evaluator.py:241-371): the reference calls
// cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) from the network pose on ALL selected correspondences, i.e.
// LM on the reprojection error (at most 20 iterations in OpenCV's cvFindExtrinsicCameraParams2).  Same compaction and
// LM as pnp_ransac_kernel, no sampling.  < 4 correspondences -> the initial pose unchanged (gdrn_evaluator.py:355-358).
__global__ void __launch_bounds__(PR_THREADS)
pnp_iterative_kernel(const PnpParams p, const float* __restrict__ rot0, const float* __restrict__ trans0) {
  extern __shared__ float sm_f[];
  float* s3 = sm_f;
  float* s2 = s3 + 3 * PR_MAX_PTS;
  unsigned short* s_src = reinterpret_cast<unsigned short*>(s2 + 2 * PR_MAX_PTS);
  __shared__ double s_red[PR_THREADS / 32][28];
  __shared__ double s_pose[12], s_save[12], s_K[9], s_step[8];
  __shared__ float s_mm[2];
  __shared__ int s_count, s_scan[PR_THREADS / 32 + 1];
  const PnpShared sh = {s3, s2, s_src, s_red, s_K, s_step, s_mm, &s_count, s_scan};

  const int roi = blockIdx.x;
  const int tid = threadIdx.x;
  if (tid < 9) s_K[tid] = (double)p.Ks[roi * 9 + tid];
  if (tid < 12) s_pose[tid] = (tid & 3) == 3 ? (double)trans0[roi * 3 + (tid >> 2)] : (double)rot0[roi * 9 + (tid >> 2) * 3 + (tid & 3)];
  const int N = gather_correspondences(p, roi, sh);
  float* out = p.poses + (long long)roi * 12;
  if (N < 4) {
    if (tid < 12) out[tid] = (float)s_pose[tid];   // exact: the pose came in as float
    if (tid == 0 && p.n_inliers) p.n_inliers[roi] = 0;
    return;
  }
  lm_refine<true>(s_pose, s_save, nullptr, N, PNP_ITERATIVE_MAX_ITERS, sh);
  if (tid < 12) out[tid] = (float)s_pose[tid];
  if (tid == 0 && p.n_inliers) p.n_inliers[roi] = N;
}

// The rules the reference's process_net_and_pnp applies after cv2.solvePnPRansac(EPNP, useExtrinsicGuess=True), one
// thread per ROI on the pose pnp_ransac_kernel wrote:
//   * < 4 correspondences or no RANSAC model (the -100 sentinel) -> the network pose (cv2 hands the guess back);
//   * net_ransac_pnp: ||t_pnp - t_net|| > 1 -> t = t_net, R stays the PnP rotation;
//   * net_ransac_pnp_rot: t = t_net always.
__global__ void pnp_net_select_kernel(float* __restrict__ poses, const float* __restrict__ rot_net,
                                      const float* __restrict__ trans_net, int n, int pnp_type) {
  const int roi = blockIdx.x * blockDim.x + threadIdx.x;
  if (roi >= n) return;
  float* P = poses + (long long)roi * 12;
  const float* tn = trans_net + roi * 3;
  if (P[0] == -100.f) {   // a rotation entry is never -100: this is the sentinel
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) P[r * 4 + c] = rot_net[roi * 9 + r * 3 + c];
      P[r * 4 + 3] = tn[r];
    }
    return;
  }
  bool use_net_t = pnp_type == PNP_NET_RANSAC_ROT;
  if (!use_net_t) {
    const double dx = (double)P[3] - tn[0], dy = (double)P[7] - tn[1], dz = (double)P[11] - tn[2];
    use_net_t = sqrt(dx * dx + dy * dy + dz * dz) > 1.0;   // gdrn_evaluator.py:347-351
  }
  if (use_net_t) { P[3] = tn[0]; P[7] = tn[1]; P[11] = tn[2]; }
}

constexpr size_t PR_SMEM = (size_t)PR_MAX_PTS * (5 * sizeof(float) + sizeof(unsigned short) + 1);

int launch_pnp(const PnpParams& p, int n, cudaStream_t st) {
  GDRN_OPT_IN_SMEM(pnp_ransac_kernel, PR_SMEM);
  pnp_ransac_kernel<<<n, PR_THREADS, PR_SMEM, st>>>(p);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_pnp_iterative(const PnpParams& p, const float* rot0, const float* trans0, int n, cudaStream_t st) {
  GDRN_OPT_IN_SMEM(pnp_iterative_kernel, PR_SMEM);
  pnp_iterative_kernel<<<n, PR_THREADS, PR_SMEM, st>>>(p, rot0, trans0);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

}  // namespace

extern "C" int gdrn_pnp_ransac_maps(const float* coor_x, const float* coor_y, const float* coor_z, const float* mask,
                                    const float* roi_coord_2d, const float* im_hw, const float* extents, const float* Ks,
                                    const int* idxs, int n, int hw, int iters, float mask_thr, float reproj_thr,
                                    unsigned seed, float* poses, int* n_inliers, unsigned char* inlier_mask, void* stream) {
  GDRN_REQUIRE(coor_x && coor_y && coor_z && mask && roi_coord_2d && im_hw && extents && Ks && poses, "pnp_ransac: null argument");
  GDRN_REQUIRE(n > 0 && hw > 0 && hw * hw <= PR_MAX_PTS, "pnp_ransac: need n > 0 and hw*hw <= 4096");
  GDRN_REQUIRE(iters >= 1 && iters <= PR_MAX_HYP, "pnp_ransac: iters must be in [1, 256]");
  PnpParams p = {};
  p.coor_x = coor_x; p.coor_y = coor_y; p.coor_z = coor_z; p.mask = mask; p.coord2d = roi_coord_2d; p.im_hw = im_hw;
  p.extents = extents; p.Ks = Ks; p.idxs = idxs; p.npts = hw * hw; p.iters = iters; p.mask_thr = mask_thr;
  p.reproj_thr = reproj_thr; p.seed = seed; p.poses = poses; p.n_inliers = n_inliers; p.inlier_mask = inlier_mask;
  return launch_pnp(p, n, (cudaStream_t)stream);
}

extern "C" int gdrn_pnp_ransac_points(const float* pts3d, const float* pts2d, const float* Ks, const int* idxs, int n,
                                      int npts, int iters, float reproj_thr, unsigned seed, float* poses, int* n_inliers,
                                      unsigned char* inlier_mask, void* stream) {
  GDRN_REQUIRE(pts3d && pts2d && Ks && poses, "pnp_ransac: null argument");
  GDRN_REQUIRE(n > 0 && npts >= 1 && npts <= PR_MAX_PTS, "pnp_ransac: need n > 0 and 1 <= npts <= 4096");
  GDRN_REQUIRE(iters >= 1 && iters <= PR_MAX_HYP, "pnp_ransac: iters must be in [1, 256]");
  PnpParams p = {};
  p.pts3d = pts3d; p.pts2d = pts2d; p.Ks = Ks; p.idxs = idxs; p.npts = npts; p.iters = iters; p.reproj_thr = reproj_thr;
  p.seed = seed; p.poses = poses; p.n_inliers = n_inliers; p.inlier_mask = inlier_mask;
  return launch_pnp(p, n, (cudaStream_t)stream);
}

extern "C" int gdrn_pnp_ransac_trace(const float* coor_x, const float* coor_y, const float* coor_z, const float* mask,
                                     const float* roi_coord_2d, const float* im_hw, const float* extents,
                                     const float* pts3d, const float* pts2d, const float* Ks, const int* idxs, int n,
                                     int npts, int iters, float mask_thr, float reproj_thr, unsigned seed, float* poses,
                                     int* n_inliers, unsigned char* inlier_mask, int* tr_count, int* tr_src,
                                     int* tr_samples, int* tr_nsol, double* tr_hyp, int* tr_cnt, int* tr_best,
                                     unsigned char* tr_inl, double* tr_round_pose, double* tr_round_cost,
                                     double* tr_pose, void* stream) {
  const bool maps = pts3d == nullptr;
  GDRN_REQUIRE(Ks && poses && (maps ? (coor_x && coor_y && coor_z && mask && roi_coord_2d && im_hw && extents) : pts2d != nullptr),
               "pnp_ransac_trace: null argument");
  GDRN_REQUIRE(tr_count && tr_src && tr_samples && tr_nsol && tr_hyp && tr_cnt && tr_best && tr_inl && tr_round_pose &&
               tr_round_cost && tr_pose, "pnp_ransac_trace: null trace buffer");
  GDRN_REQUIRE(n > 0 && npts >= 1 && npts <= PR_MAX_PTS, "pnp_ransac_trace: need n > 0 and 1 <= npts <= 4096");
  GDRN_REQUIRE(iters >= 1 && iters <= PR_MAX_HYP, "pnp_ransac_trace: iters must be in [1, 256]");
  PnpParams p = {};
  if (maps) {
    p.coor_x = coor_x; p.coor_y = coor_y; p.coor_z = coor_z; p.mask = mask; p.coord2d = roi_coord_2d; p.im_hw = im_hw;
    p.extents = extents; p.mask_thr = mask_thr;
  } else {
    p.pts3d = pts3d; p.pts2d = pts2d;
  }
  p.Ks = Ks; p.idxs = idxs; p.npts = npts; p.iters = iters; p.reproj_thr = reproj_thr; p.seed = seed; p.poses = poses;
  p.n_inliers = n_inliers; p.inlier_mask = inlier_mask;
  p.tr = {tr_count, tr_src, tr_samples, tr_nsol, tr_hyp, tr_cnt, tr_best, tr_inl, tr_round_pose, tr_round_cost, tr_pose};
  return launch_pnp(p, n, (cudaStream_t)stream);
}

extern "C" int gdrn_pnp_net_maps(const float* coor_x, const float* coor_y, const float* coor_z, const float* mask,
                                 const float* roi_coord_2d, const float* im_hw, const float* extents, const float* Ks,
                                 const float* rot_net, const float* trans_net, int n, int hw, int pnp_type, float mask_thr,
                                 float reproj_thr, int ransac_iters, unsigned seed, float* poses, int* n_used, void* stream) {
  GDRN_REQUIRE(coor_x && coor_y && coor_z && mask && roi_coord_2d && im_hw && extents && Ks && rot_net && trans_net && poses,
               "pnp_net: null argument");
  GDRN_REQUIRE(n > 0 && hw > 0 && hw * hw <= PR_MAX_PTS, "pnp_net: need n > 0 and hw*hw <= 4096");
  GDRN_REQUIRE(pnp_type == PNP_NET_ITER || pnp_type == PNP_NET_RANSAC || pnp_type == PNP_NET_RANSAC_ROT,
               "pnp_net: pnp_type must be 0 (net_iter_pnp), 1 (net_ransac_pnp) or 2 (net_ransac_pnp_rot)");
  GDRN_REQUIRE(pnp_type == PNP_NET_ITER || (ransac_iters >= 1 && ransac_iters <= PR_MAX_HYP),
               "pnp_net: ransac_iters must be in [1, 256]");
  cudaStream_t st = (cudaStream_t)stream;
  PnpParams p = {};
  p.coor_x = coor_x; p.coor_y = coor_y; p.coor_z = coor_z; p.mask = mask; p.coord2d = roi_coord_2d; p.im_hw = im_hw;
  p.extents = extents; p.Ks = Ks; p.npts = hw * hw; p.iters = ransac_iters; p.mask_thr = mask_thr;
  p.reproj_thr = reproj_thr; p.seed = seed; p.poses = poses; p.n_inliers = n_used;
  if (pnp_type == PNP_NET_ITER) return launch_pnp_iterative(p, rot_net, trans_net, n, st);
  const int rc = launch_pnp(p, n, st);
  if (rc != GDRN_OK) return rc;
  pnp_net_select_kernel<<<(n + 127) / 128, 128, 0, st>>>(poses, rot_net, trans_net, n, pnp_type);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_pnp_iterative_points(const float* pts3d, const float* pts2d, const float* Ks, const float* rot0,
                                         const float* trans0, int n, int npts, float* poses, void* stream) {
  GDRN_REQUIRE(pts3d && pts2d && Ks && rot0 && trans0 && poses, "pnp_iterative: null argument");
  GDRN_REQUIRE(n > 0 && npts >= 1 && npts <= PR_MAX_PTS, "pnp_iterative: need n > 0 and 1 <= npts <= 4096");
  PnpParams p = {};
  p.pts3d = pts3d; p.pts2d = pts2d; p.Ks = Ks; p.npts = npts; p.iters = 1; p.poses = poses;
  return launch_pnp_iterative(p, rot0, trans0, n, (cudaStream_t)stream);
}
