/* ORACLE (test infrastructure, NOT product code): CPU restatements of the reference's native ops.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library.  Build: oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp).
 *
 * Each function cites the reference lines it follows (paths relative to the reference tree).
 * Where the reference is CUDA built with nvcc's default --fmad=true, the fused-multiply-add placement
 * that ptxas 12.9 produces for sm_90a (inspected in the SASS of the reference file compiled for sm_90a)
 * is written out with fmaf() so the results are bit-identical to that build.  Pinned against what the
 * real reference computes (tests/golden/: FPS from the reference .cpp, voting/nnd/flow from the reference
 * .cu built for sm_90a and run on an H100, tools/make_golden_ref.py).
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------------
 * Farthest point sampling: core/csrc/fps/src/farthest_point_sampling.cpp:40-160.
 * start < 0  -> init_center variant (:118-160); start >= 0 -> explicit first index (the random-start
 * variant :76-104 with cur_idx given instead of rand()%pn).
 * ---------------------------------------------------------------------------------------------- */
static float sqnorm3(float x, float y, float z) { return x * x + y * y + z * z; }

static int find_max_idx(const float* min_dist, const unsigned char* mask, int pn) {
  int max_idx = 0;
  float max_d = 0.f;
  for (int i = 0; i < pn; i++) {
    if (mask[i]) continue;
    if (min_dist[i] > max_d) { max_idx = i; max_d = min_dist[i]; }
  }
  return max_idx;
}

void oracle_fps(const float* pts, int* idxs, int pn, int sn, int start) {
  unsigned char* mask = (unsigned char*)calloc(pn, 1);
  float* min_dist = (float*)malloc(sizeof(float) * pn);
  for (int i = 0; i < pn; i++) min_dist[i] = FLT_MAX;
  int cur;
  if (start < 0) {
    float mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX}, mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
    for (int i = 0; i < pn; i++)
      for (int k = 0; k < 3; k++) {
        float v = pts[i * 3 + k];
        if (v > mx[k]) mx[k] = v;
        if (v < mn[k]) mn[k] = v;
      }
    float c[3];
    for (int k = 0; k < 3; k++) c[k] = (mx[k] + mn[k]) * (1.f / 2.f);
    for (int i = 0; i < pn; i++) {
      float d = sqnorm3(pts[i * 3] - c[0], pts[i * 3 + 1] - c[1], pts[i * 3 + 2] - c[2]);
      if (d < min_dist[i]) min_dist[i] = d;
    }
    cur = find_max_idx(min_dist, mask, pn);
  } else {
    cur = start;
  }
  for (int s = 0; s < sn; s++) {
    mask[cur] = 1;
    idxs[s] = cur;
    if (s < sn - 1) {
      for (int i = 0; i < pn; i++) {
        if (mask[i]) continue;
        float d = sqnorm3(pts[i * 3] - pts[cur * 3], pts[i * 3 + 1] - pts[cur * 3 + 1], pts[i * 3 + 2] - pts[cur * 3 + 2]);
        if (d < min_dist[i]) min_dist[i] = d;
      }
      cur = find_max_idx(min_dist, mask, pn);
    }
  }
  free(mask);
  free(min_dist);
}

/* ------------------------------------------------------------------------------------------------
 * RANSAC voting: core/csrc/ransac_voting/src/ransac_voting_kernel.cu
 * ---------------------------------------------------------------------------------------------- */
/* :11-49 */
void oracle_generate_hypothesis(const float* direct, const float* coords, const int* idxs, float* hypo, int tn, int vn,
                                int hn) {
  (void)tn;
#pragma omp parallel for
  for (int hvi = 0; hvi < hn * vn; hvi++) {
    int vi = hvi % vn;
    int t0 = idxs[hvi * 2], t1 = idxs[hvi * 2 + 1];
    float d0x = direct[(t0 * vn + vi) * 2], d0y = direct[(t0 * vn + vi) * 2 + 1];
    float d1x = direct[(t1 * vn + vi) * 2], d1y = direct[(t1 * vn + vi) * 2 + 1];
    float cx0 = coords[t0 * 2], cy0 = coords[t0 * 2 + 1], cx1 = coords[t1 * 2], cy1 = coords[t1 * 2 + 1];
    /* nx = d.y, ny = -d.x */
    float a = d0x * d1y, b = d0y * d1x;
    float det_y = b - a; /* nx1*ny0 - nx0*ny1 */
    if (fabs((double)fabsf(det_y)) < 1e-6) continue;
    float det_x = a - b; /* ny1*nx0 - ny0*nx1 */
    if (fabs((double)fabsf(det_x)) < 1e-6) continue;
    float s1 = fmaf(d1y, cx1, -(d1x * cy1));
    float s0 = fmaf(d0y, cx0, -(d0x * cy0));
    float num_y = fmaf(d1y, s0, -(d0y * s1));
    float num_x = fmaf(-d1x, s0, d0x * s1);
    hypo[hvi * 2] = num_x / det_x;
    hypo[hvi * 2 + 1] = num_y / det_y;
  }
}

/* :170-229 */
void oracle_generate_hypothesis_vp(const float* direct, const float* coords, const int* idxs, float* hypo, int tn, int vn,
                                   int hn) {
  (void)tn;
#pragma omp parallel for
  for (int hvi = 0; hvi < hn * vn; hvi++) {
    int vi = hvi % vn;
    int id0 = idxs[hvi * 2], id1 = idxs[hvi * 2 + 1];
    float dx0 = direct[(id0 * vn + vi) * 2], dy0 = direct[(id0 * vn + vi) * 2 + 1];
    float dx1 = direct[(id1 * vn + vi) * 2], dy1 = direct[(id1 * vn + vi) * 2 + 1];
    float cx0 = coords[id0 * 2], cy0 = coords[id0 * 2 + 1], cx1 = coords[id1 * 2], cy1 = coords[id1 * 2 + 1];
    float lz0 = fmaf(dx0, cy0, -(dy0 * cx0));
    float lz1 = fmaf(dx1, cy1, -(dy1 * cx1));
    float x = fmaf(dx1, lz0, -(dx0 * lz1));
    float y = fmaf(dy1, lz0, -(dy0 * lz1));
    float z = fmaf(dx0, dy1, -(dy0 * dx1));
    float vx0 = dx0 * fmaf(-cx0, z, x), vx1 = dx1 * fmaf(-cx1, z, x);
    float vy0 = dy0 * fmaf(-cy0, z, y), vy1 = dy1 * fmaf(-cy1, z, y);
    if (vx0 < 0 && vx1 < 0 && vy0 < 0 && vy1 < 0) { x = -x; y = -y; z = -z; }
    if (vx0 * vx1 < 0 || vy0 * vy1 < 0) { x = 0.f; y = 0.f; z = 0.f; }
    hypo[hvi * 3] = x;
    hypo[hvi * 3 + 1] = y;
    hypo[hvi * 3 + 2] = z;
  }
}

/* :88-126 and :268-310 ; inliers is in/out ([hn,vn,tn] u8), counts (optional) [hn,vn] = number of 1s written */
void oracle_voting(const float* direct, const float* coords, const float* hypo, unsigned char* inliers, int* counts,
                   int tn, int vn, int hn, float thresh, int vanishing_point) {
  const int HD = vanishing_point ? 3 : 2;
#pragma omp parallel for
  for (int hi = 0; hi < hn; hi++) {
    for (int vi = 0; vi < vn; vi++) {
      int cnt = 0;
      const float hx = hypo[(hi * vn + vi) * HD], hy = hypo[(hi * vn + vi) * HD + 1];
      const float hz = vanishing_point ? hypo[(hi * vn + vi) * HD + 2] : 0.f;
      for (int ti = 0; ti < tn; ti++) {
        float cx = coords[ti * 2], cy = coords[ti * 2 + 1];
        float nx = direct[(ti * vn + vi) * 2], ny = direct[(ti * vn + vi) * 2 + 1];
        float dx, dy;
        if (vanishing_point) { dx = fmaf(-cx, hz, hx); dy = fmaf(-cy, hz, hy); }
        else { dx = hx - cx; dy = hy - cy; }
        float norm1 = sqrtf(fmaf(nx, nx, ny * ny));
        float norm2 = sqrtf(fmaf(dx, dx, dy * dy));
        if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) continue;
        float den = norm1 * norm2;
        int in;
        if (vanishing_point) {
          float vx = nx * dx, vy = ny * dy;
          float ang = (vx + vy) / den;
          if (vx < 0 || vy < 0) continue;
          in = fabsf(ang) > thresh;
        } else {
          float ang = fmaf(nx, dx, ny * dy) / den;
          in = ang > thresh;
        }
        if (in) {
          if (inliers) inliers[((size_t)hi * vn + vi) * tn + ti] = 1;
          cnt++;
        }
      }
      if (counts) counts[hi * vn + vi] = cnt;
    }
  }
}

/* ------------------------------------------------------------------------------------------------
 * Chamfer / NN distance forward: core/csrc/torch_nndistance/src/nnd_cuda_kernel.cu:8-130
 * (d = fma(dz,dz, fma(dx,dx, dy*dy)); lowest index on ties).  The CPU twin in the reference
 * (nnd_cpu.cpp:3-25) accumulates in double and is NOT what the CUDA build computes.
 * ---------------------------------------------------------------------------------------------- */
void oracle_nnd_forward(const float* a, const float* b, float* dist, int* idx, int bs, int n, int m) {
#pragma omp parallel for collapse(2)
  for (int i = 0; i < bs; i++)
    for (int j = 0; j < n; j++) {
      float x1 = a[(i * n + j) * 3], y1 = a[(i * n + j) * 3 + 1], z1 = a[(i * n + j) * 3 + 2];
      float best = 0.f;
      int best_i = 0;
      for (int k = 0; k < m; k++) {
        float x2 = b[(i * m + k) * 3] - x1, y2 = b[(i * m + k) * 3 + 1] - y1, z2 = b[(i * m + k) * 3 + 2] - z1;
        float d = fmaf(z2, z2, fmaf(x2, x2, y2 * y2));
        if (k == 0 || d < best) { best = d; best_i = k; }
      }
      dist[i * n + j] = best;
      idx[i * n + j] = best_i;
    }
}

/* backward: nnd_cuda_kernel.cu:164-183 (one direction; accumulates) */
void oracle_nnd_backward(const float* a, const float* b, const float* grad_dist, const int* idx, float* grad_a,
                         float* grad_b, int bs, int n, int m) {
  for (int i = 0; i < bs; i++)
    for (int j = 0; j < n; j++) {
      int j2 = idx[i * n + j];
      float g = grad_dist[i * n + j] * 2;
      for (int c = 0; c < 3; c++) {
        float v = g * (a[(i * n + j) * 3 + c] - b[(i * m + j2) * 3 + c]);
        grad_a[(i * n + j) * 3 + c] += v;
        grad_b[(i * m + j2) * 3 + c] += -v;
      }
    }
}

/* ------------------------------------------------------------------------------------------------
 * Flow: core/csrc/flow/src/flow_cuda_kernel.cu:26-65 (float instantiation)
 * ---------------------------------------------------------------------------------------------- */
void oracle_flow(const float* depth_src, const float* depth_tgt, const float* KT, const float* Kinv, float* flow,
                 float* valid, int batch, int height, int width) {
  const long hw = (long)height * width;
#pragma omp parallel for
  for (long index = 0; index < hw * batch; index++) {
    int w = (int)(index % width), h = (int)((index / width) % height), b = (int)(index / hw);
    float d = depth_src[index];
    float f0 = 0.f, f1 = 0.f, ok = 0.f;
    if ((double)d > 1E-3) {
      const float* ki = Kinv + b * 9;
      const float* kt = KT + b * 12;
      float wf = (float)w, hf = (float)h;
      float x = (fmaf(wf, ki[0], hf * ki[1]) + ki[2]) * d;
      float y = (fmaf(wf, ki[3], hf * ki[4]) + ki[5]) * d;
      float xp = fmaf(d, kt[2], fmaf(x, kt[0], y * kt[1])) + kt[3];
      float yp = fmaf(d, kt[6], fmaf(x, kt[4], y * kt[5])) + kt[7];
      float zs = fmaf(d, kt[10], fmaf(x, kt[8], y * kt[9])) + kt[11];
      float zp = (float)((double)zs + 1E-15);
      float wp = xp / zp, hp = yp / zp;
      if (wp >= 0.f && wp <= (float)(width - 1) && hp >= 0.f && hp <= (float)(height - 1)) {
        int wi = (int)roundf(wp), hi = (int)roundf(hp);
        float dt = depth_tgt[((long)b * height + hi) * width + wi];
        if ((double)fabsf(zp - dt) < 3E-3) { f0 = hp - hf; f1 = wp - wf; ok = 1.f; }
      }
    }
    flow[((long)b * 2 + 0) * hw + (long)h * width + w] = f0;
    flow[((long)b * 2 + 1) * hw + (long)h * width + w] = f1;
    valid[index] = ok;
  }
}

/* =================================================================================================
 * ROI crop + resize = cv2.warpAffine(img, trans, (ow, oh), flags=INTER_LINEAR | INTER_NEAREST), borderMode constant 0,
 * as called by crop_resize_by_warp_affine (core/utils/data_utils.py:115-133; predictor_gdrn.py:417-438).
 * The arithmetic lives in OpenCV 4.x (un-vendored dependency, opencv-python; imgwarp.cpp warpAffine / WarpAffineInvoker /
 * remapBilinear): the forward matrix is inverted in double, destination pixels are mapped to source coordinates in
 * 10-bit fixed point (per-column terms cvRound(M0*x*1024), per-row terms cvRound((M1*y+M2)*1024) + round_delta),
 * bilinear: 5 fractional bits, uint8 data blended with 15-bit integer weights ((1-fx)(1-fy) ... scaled by 32768,
 * saturated to short with the deficit added to the fx*fy weight -> (32767, 0, 0, 1) at integer positions),
 * result (sum + 16384) >> 15; float data blended with the float weights; taps outside the image read 0.
 * Pinned bit-exactly (uint8, nearest) / to 1e-6 (float bilinear) against cv2 itself in tests/test_oracle_pinning.py.
 * ================================================================================================= */
static int ora_cvround(double v) {
  double r = nearbyint(v); /* round half to even (default rounding mode), like cvRound / lrint */
  if (r > 2147483647.0) return 2147483647;
  if (r < -2147483648.0) return (-2147483647 - 1);
  return (int)r;
}

/* forward 2x3 matrix (src -> dst) to the inverse used for sampling: cv::warpAffine, "if( !(flags & WARP_INVERSE_MAP) )" */
void oracle_invert_affine(const double* M, double* iM) {
  double D = M[0] * M[4] - M[1] * M[3];
  D = D != 0 ? 1. / D : 0;
  double A11 = M[4] * D, A22 = M[0] * D;
  iM[0] = A11; iM[1] = M[1] * (-D); iM[3] = M[3] * (-D); iM[4] = A22;
  double b1 = -iM[0] * M[2] - iM[1] * M[5];
  double b2 = -iM[3] * M[2] - iM[4] * M[5];
  iM[2] = b1; iM[5] = b2;
}

static void ora_src_coord(const double* iM, int x, int y, int nearest, int* X, int* Y) {
  const int AB_BITS = 10, AB_SCALE = 1 << 10, INTER_BITS = 5;
  const int round_delta = nearest ? AB_SCALE / 2 : AB_SCALE / 32 / 2;
  const int adelta = ora_cvround(iM[0] * x * AB_SCALE), bdelta = ora_cvround(iM[3] * x * AB_SCALE);
  const int X0 = ora_cvround((iM[1] * y + iM[2]) * AB_SCALE) + round_delta;
  const int Y0 = ora_cvround((iM[4] * y + iM[5]) * AB_SCALE) + round_delta;
  if (nearest) { *X = (X0 + adelta) >> AB_BITS; *Y = (Y0 + bdelta) >> AB_BITS; }
  else { *X = (X0 + adelta) >> (AB_BITS - INTER_BITS); *Y = (Y0 + bdelta) >> (AB_BITS - INTER_BITS); }
}

static void ora_bilinear_itab(int fx, int fy, int* w) {
  /* float table entries are exact multiples of 1/1024; x 32768 is exact; saturate_cast<short> clips 32768 -> 32767 */
  const float ax = fx * (1.f / 32), ay = fy * (1.f / 32);
  const float t[4] = {(1.f - ay) * (1.f - ax), (1.f - ay) * ax, ay * (1.f - ax), ay * ax};
  int isum = 0;
  for (int k = 0; k < 4; ++k) {
    int r = ora_cvround((double)(t[k] * 32768.f));
    if (r > 32767) r = 32767;
    w[k] = r; isum += r;
  }
  if (isum != 32768) w[3] -= (isum - 32768);   /* only element (1,1) is inspected for ksize = 2 */
}

/* uint8 image [H][W][C] -> dst [oh][ow][C] */
void oracle_warp_affine_u8(const unsigned char* src, int H, int W, int C, const double* M, unsigned char* dst, int oh, int ow) {
  double iM[6];
  oracle_invert_affine(M, iM);
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      int X, Y, w[4];
      ora_src_coord(iM, x, y, 0, &X, &Y);
      int sx = X >> 5, sy = Y >> 5;
      if (sx > 32767) sx = 32767; if (sx < -32768) sx = -32768;   /* saturate_cast<short> */
      if (sy > 32767) sy = 32767; if (sy < -32768) sy = -32768;
      ora_bilinear_itab(X & 31, Y & 31, w);
      for (int c = 0; c < C; ++c) {
        int v = 0;
        for (int k = 0; k < 4; ++k) {
          const int xx = sx + (k & 1), yy = sy + (k >> 1);
          const int s = (xx >= 0 && xx < W && yy >= 0 && yy < H) ? src[((long long)yy * W + xx) * C + c] : 0;
          v += s * w[k];
        }
        v = (v + (1 << 14)) >> 15;
        dst[((long long)y * ow + x) * C + c] = (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
      }
    }
}

/* float image [H][W][C]; nearest = 1: INTER_NEAREST */
void oracle_warp_affine_f32(const float* src, int H, int W, int C, const double* M, float* dst, int oh, int ow, int nearest) {
  double iM[6];
  oracle_invert_affine(M, iM);
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      int X, Y;
      ora_src_coord(iM, x, y, nearest, &X, &Y);
      if (nearest) {
        for (int c = 0; c < C; ++c)
          dst[((long long)y * ow + x) * C + c] = (X >= 0 && X < W && Y >= 0 && Y < H) ? src[((long long)Y * W + X) * C + c] : 0.f;
        continue;
      }
      int sx = X >> 5, sy = Y >> 5;
      const float ax = (X & 31) * (1.f / 32), ay = (Y & 31) * (1.f / 32);
      const float w[4] = {(1.f - ay) * (1.f - ax), (1.f - ay) * ax, ay * (1.f - ax), ay * ax};
      for (int c = 0; c < C; ++c) {
        float s[4];
        for (int k = 0; k < 4; ++k) {
          const int xx = sx + (k & 1), yy = sy + (k >> 1);
          s[k] = (xx >= 0 && xx < W && yy >= 0 && yy < H) ? src[((long long)yy * W + xx) * C + c] : 0.f;
        }
        dst[((long long)y * ow + x) * C + c] = s[0] * w[0] + s[1] * w[1] + s[2] * w[2] + s[3] * w[3];
      }
    }
}
