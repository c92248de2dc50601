// GDRN training loss on the GPU: the coordinate, mask, full-mask and region terms over the head's 64x64 maps,
// symmetry-aware point matching and the centroid / z terms, with their gradients, in four forward launches and one
// backward launch with no host synchronisation between them.
//
// Replaces GDRN_DoubleMask.gdrn_loss (core/gdrn_modeling/models/GDRN_double_mask.py:287-536), PyPMLoss
// (core/gdrn_modeling/losses/pm_loss.py) and get_closest_rot_batch (core/utils/pose_utils.py:472-528).  DESIGN.md §7r
// pins every rule.
//   1. gl_dense_kernel     (pixel tile, ROI): the three L1 coordinate sums, the two mask sums, the region
//      cross-entropy (online log-sum-exp over the R+1 logits, one read of each), the two mask counts and the label
//      check, as one fixed-order f64 partial per CTA; each pixel's log-sum-exp is kept for the backward.
//   2. gl_pm_kernel        one CTA per ROI: the closest symmetric GT rotation by an (error, index) argmin over R_gt
//      and R_gt S_k, then sum |w (R_est - R_gt') p| and the nine sums sign(.) w p^T over the points.
//   3. gl_finalize_kernel  one CTA: partials in a fixed order in f64 -> normalisers, weighted losses, error flag.
//   4. gl_backward_kernel  (pixel tile, ROI): every map gradient, scaled by the upstream gradients; CTA (0, 0) also
//      writes the rotation, centroid and z gradients from the stored sums.
// The per-pixel products and differences use round-to-nearest intrinsics, so no FMA contraction makes them differ
// from an fp32 restatement of the same expressions.
#include "common.cuh"

namespace {

constexpr int GL_THREADS = 128;
constexpr int GL_VEC = 4;                         // pixels per thread
constexpr int GL_TILE = GL_THREADS * GL_VEC;      // pixels per CTA
constexpr int GL_PM_THREADS = 256;
constexpr int GL_NPART = 8;                       // xyz x, y, z, mask, full mask, region CE, count xyz, count region
constexpr int GL_NRES = 10;                       // 9 losses + error flag
constexpr int GL_NOFF = 10;

// inputs (host array of device pointers), in this order
enum {
  IN_OUT_X, IN_OUT_Y, IN_OUT_Z, IN_OUT_MASK, IN_OUT_FULL,   // [B,1,H,W] f32, batch stride given, plane contiguous
  IN_M_XYZ, IN_M_MASK, IN_M_FULL, IN_M_REGION,              // [B,H,W] f32 (the selected GT masks)
  IN_GT_XYZ, IN_OUT_REGION, IN_GT_REGION,                   // [B,3,H,W] f32, [B,R1,H,W] f32, [B,H,W] i64
  IN_OUT_ROT, IN_GT_ROT, IN_POINTS, IN_EXTENTS,             // [B,3,3], [B,3,3], [B,N,3], [B,3] f32
  IN_SYM_TABLE, IN_SYM_RANGE,                               // [T,3,3] f32, [B,2] i32 (first row, count)
  IN_OUT_CENTROID, IN_OUT_TZ, IN_GT_RATIO, IN_GT_TRANS,     // [B,2], [B], [B,3], [B,3] f32
  IN_COUNT
};
// terms (flags bits)
enum { F_GEO = 1, F_FULL = 2, F_MASK_BCE = 4, F_FULL_BCE = 8, F_PM = 16, F_PM_EXTENT = 32, F_CENTROID = 64, F_Z = 128,
       F_Z_ABS = 256 };
// loss weights (params), and the result / upstream-gradient slots
enum { W_XYZ, W_MASK, W_FULL, W_REGION, W_PM, W_CENTROID, W_Z, W_COUNT };
enum { R_X, R_Y, R_Z, R_MASK, R_FULL, R_REGION, R_PM, R_CENTROID, R_TZ, R_ERR };
// gradient outputs (host array of device pointers)
enum { G_X, G_Y, G_Z, G_MASK, G_FULL, G_REGION, G_ROT, G_CENTROID, G_TZ, G_COUNT };

struct GlArgs {
  const void* in[IN_COUNT];
  long long bs[5];   // batch strides (elements) of the five single-plane head outputs
  float w[W_COUNT];
  int B, HW, R1, N, flags, tiles;
};

inline size_t gl_align(size_t x) { return (x + 255) & ~(size_t)255; }
inline int gl_tiles(int HW) { return (HW + GL_TILE - 1) / GL_TILE; }

struct GlLayout {
  size_t off[GL_NOFF + 1];
};

GlLayout gl_layout(int B, int HW) {
  const size_t P = (size_t)B * gl_tiles(HW);
  const size_t sz[GL_NOFF] = {
      P * GL_NPART * 8,        // 0 partial [P,8] f64
      P * 4,                   // 1 partial_err [P] i32
      (size_t)B * HW * 4,      // 2 lse [B,HW] f32 (region log-sum-exp per pixel)
      (size_t)B * 4,           // 3 sym_idx [B] i32 (-1 = R_gt itself, k = R_gt S_k)
      (size_t)B * 9 * 4,       // 4 rot_sel [B,3,3] f32 (R_gt')
      (size_t)B * 8,           // 5 pm_abs [B] f64
      (size_t)B * 9 * 8,       // 6 pm_sign [B,3,3] f64
      (size_t)B * 4,           // 7 sym_err [B] f32 (the chosen candidate's error, degrees)
      4 * 4,                   // 8 norm [4] f32
      GL_NRES * 4,             // 9 result [10] f32
  };
  GlLayout l;
  size_t o = 0;
  for (int i = 0; i < GL_NOFF; ++i) {
    l.off[i] = o;
    o = gl_align(o + sz[i]);
  }
  l.off[GL_NOFF] = o;
  return l;
}

struct GlWs {
  double* partial;
  int* partial_err;
  float* lse;
  int* sym_idx;
  float* rot_sel;
  double* pm_abs;
  double* pm_sign;
  float* sym_err;
  float* norm;
  float* result;
};

GlWs gl_ws(void* workspace, int B, int HW) {
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  const GlLayout l = gl_layout(B, HW);
  GlWs w;
  w.partial = reinterpret_cast<double*>(base + l.off[0]);
  w.partial_err = reinterpret_cast<int*>(base + l.off[1]);
  w.lse = reinterpret_cast<float*>(base + l.off[2]);
  w.sym_idx = reinterpret_cast<int*>(base + l.off[3]);
  w.rot_sel = reinterpret_cast<float*>(base + l.off[4]);
  w.pm_abs = reinterpret_cast<double*>(base + l.off[5]);
  w.pm_sign = reinterpret_cast<double*>(base + l.off[6]);
  w.sym_err = reinterpret_cast<float*>(base + l.off[7]);
  w.norm = reinterpret_cast<float*>(base + l.off[8]);
  w.result = reinterpret_cast<float*>(base + l.off[9]);
  return w;
}

template <typename T> __device__ __forceinline__ const T* gl_in(const GlArgs& a, int k) {
  return static_cast<const T*>(a.in[k]);
}

// GL_VEC consecutive pixels starting at p of a plane: one float4 when VEC (plane start and p 16-byte aligned, HW a
// multiple of 4), else scalar loads with zero past the end
template <bool VEC> __device__ __forceinline__ void gl_ld(const float* __restrict__ plane, int p, int HW, float v[GL_VEC]) {
  if (VEC) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(plane + p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j) v[j] = p + j < HW ? __ldg(plane + p + j) : 0.f;
  }
}
template <bool VEC> __device__ __forceinline__ void gl_st(float* __restrict__ plane, int p, int HW, const float v[GL_VEC]) {
  if (VEC) {
    *reinterpret_cast<float4*>(plane + p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j)
      if (p + j < HW) plane[p + j] = v[j];
  }
}

__device__ __forceinline__ float gl_sign(float d) { return (float)((d > 0.f) - (d < 0.f)); }
// BCEWithLogits(x, y) in torch's overflow-safe form
__device__ __forceinline__ float gl_bce(float x, float y) {
  return __fadd_rn(__fsub_rn(fmaxf(x, 0.f), __fmul_rn(x, y)), log1pf(expf(-fabsf(x))));
}
__device__ __forceinline__ float gl_sigmoid(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// fixed-order CTA sum of GL_NPART f64 values per thread; the result is in s[q][0]
__device__ __forceinline__ void gl_cta_sum(double (*s)[GL_THREADS], int tid) {
  __syncthreads();
  for (int h = GL_THREADS / 2; h; h >>= 1) {
    if (tid < h) {
#pragma unroll
      for (int q = 0; q < GL_NPART; ++q) s[q][tid] += s[q][tid + h];
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------- stage 1
template <bool VEC>
__global__ void __launch_bounds__(GL_THREADS) gl_dense_kernel(GlArgs a, GlWs w) {
  __shared__ double s_red[GL_NPART][GL_THREADS];
  __shared__ int s_err;
  const int b = blockIdx.y, tid = threadIdx.x, HW = a.HW;
  const int p = blockIdx.x * GL_TILE + tid * GL_VEC;
  const size_t bp = (size_t)b * HW;
  if (tid == 0) s_err = 0;
  __syncthreads();
  double acc[GL_NPART];
#pragma unroll
  for (int q = 0; q < GL_NPART; ++q) acc[q] = 0.0;
  if (p < HW) {
    float mx[GL_VEC], mm[GL_VEC], mr[GL_VEC], o[GL_VEC], g[GL_VEC];
    // coordinates: |out m - gt m| per axis
    gl_ld<VEC>(gl_in<float>(a, IN_M_XYZ) + bp, p, HW, mx);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gl_ld<VEC>(gl_in<float>(a, IN_OUT_X + c) + b * a.bs[c], p, HW, o);
      gl_ld<VEC>(gl_in<float>(a, IN_GT_XYZ) + (size_t)(3 * b + c) * HW, p, HW, g);
#pragma unroll
      for (int j = 0; j < GL_VEC; ++j) acc[c] += fabsf(__fsub_rn(__fmul_rn(o[j], mx[j]), __fmul_rn(g[j], mx[j])));
    }
    // masks: L1 or BCE-with-logits of the raw head output against the GT
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      if (f == 1 && !(a.flags & F_FULL)) break;
      const bool bce = a.flags & (f ? F_FULL_BCE : F_MASK_BCE);
      gl_ld<VEC>(gl_in<float>(a, f ? IN_OUT_FULL : IN_OUT_MASK) + b * a.bs[3 + f], p, HW, o);
      gl_ld<VEC>(gl_in<float>(a, f ? IN_M_FULL : IN_M_MASK) + bp, p, HW, mm);
#pragma unroll
      for (int j = 0; j < GL_VEC; ++j)
        if (p + j < HW) acc[3 + f] += bce ? gl_bce(o[j], mm[j]) : fabsf(__fsub_rn(o[j], mm[j]));
    }
    // region: cross-entropy of the logits out m against the label gt_region * long(m)
    gl_ld<VEC>(gl_in<float>(a, IN_M_REGION) + bp, p, HW, mr);
    const long long* lab = gl_in<long long>(a, IN_GT_REGION) + bp;
    int t[GL_VEC];
    bool bad = false;
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j) {
      const long long l = p + j < HW ? lab[p + j] * (long long)mr[j] : 0;
      bad |= l < 0 || l >= a.R1;
      t[j] = (int)l;
    }
    if (bad) s_err = 1;
    float m[GL_VEC], s[GL_VEC], xt[GL_VEC];
    const float* reg = gl_in<float>(a, IN_OUT_REGION) + (size_t)b * a.R1 * HW;
    gl_ld<VEC>(reg, p, HW, o);
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j) {
      m[j] = __fmul_rn(o[j], mr[j]);
      s[j] = 1.f;
      xt[j] = m[j];
    }
#pragma unroll 4
    for (int c = 1; c < a.R1; ++c) {
      gl_ld<VEC>(reg + (size_t)c * HW, p, HW, o);
#pragma unroll
      for (int j = 0; j < GL_VEC; ++j) {
        const float x = __fmul_rn(o[j], mr[j]);
        if (x > m[j]) {
          s[j] = __fadd_rn(__fmul_rn(s[j], expf(__fsub_rn(m[j], x))), 1.f);
          m[j] = x;
        } else {
          s[j] = __fadd_rn(s[j], expf(__fsub_rn(x, m[j])));
        }
        if (c == t[j]) xt[j] = x;
      }
    }
    float lse[GL_VEC];
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j) {
      lse[j] = __fadd_rn(m[j], logf(s[j]));
      if (p + j < HW) {
        acc[5] += __fsub_rn(lse[j], xt[j]);
        acc[6] += mx[j];
        acc[7] += mr[j];
      }
    }
    gl_st<VEC>(w.lse + bp, p, HW, lse);
  }
#pragma unroll
  for (int q = 0; q < GL_NPART; ++q) s_red[q][tid] = acc[q];
  gl_cta_sum(s_red, tid);
  if (tid < GL_NPART) {
    const size_t pi = (size_t)b * gridDim.x + blockIdx.x;
    w.partial[pi * GL_NPART + tid] = s_red[tid][0];
    if (tid == 0) w.partial_err[pi] = s_err;
  }
}

// ---------------------------------------------------------------------------------------------------------- stage 2
__device__ __forceinline__ void gl_matmul3(const float* A, const float* S, float* C) {   // C = A S, fp32
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      C[3 * i + j] = __fadd_rn(__fadd_rn(__fmul_rn(A[3 * i], S[j]), __fmul_rn(A[3 * i + 1], S[3 + j])),
                               __fmul_rn(A[3 * i + 2], S[6 + j]));
}
// pose_error.re: arccos(clamp(0.5 (trace(R_est R^T) - 1), -1, 1)) in degrees, fp32
__device__ __forceinline__ float gl_re(const float* E, const float* R) {
  float tr = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) tr = __fadd_rn(tr, __fmul_rn(E[k], R[k]));
  tr = fminf(tr, 3.f);
  const float c = fminf(1.f, fmaxf(-1.f, __fmul_rn(0.5f, __fsub_rn(tr, 1.f))));
  return __fmul_rn(acosf(c), 57.29577951308232f);
}
__device__ __forceinline__ bool gl_better(float e, int i, float e2, int i2) { return e < e2 || (e == e2 && i < i2); }

__global__ void __launch_bounds__(GL_PM_THREADS) gl_pm_kernel(GlArgs a, GlWs w) {
  constexpr int NW = GL_PM_THREADS / 32;
  __shared__ float s_e[NW];
  __shared__ int s_i[NW];
  __shared__ float s_rot[9];
  __shared__ double s_acc[10][NW];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float E[9], G[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    E[k] = gl_in<float>(a, IN_OUT_ROT)[(size_t)b * 9 + k];
    G[k] = gl_in<float>(a, IN_GT_ROT)[(size_t)b * 9 + k];
  }
  const int* range = gl_in<int>(a, IN_SYM_RANGE);
  const int k0 = range ? range[2 * b] : 0, K = range ? range[2 * b + 1] : 0;
  const float* table = gl_in<float>(a, IN_SYM_TABLE);
  // candidate -1 is R_gt itself; the reference's strict < keeps the earliest candidate on a tie
  float be = tid == 0 ? gl_re(E, G) : INFINITY;
  int bi = tid == 0 ? -1 : 0x7fffffff;
  for (int k = tid; k < K; k += GL_PM_THREADS) {
    float S[9], C[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) S[q] = table[(size_t)(k0 + k) * 9 + q];
    gl_matmul3(G, S, C);
    const float e = gl_re(E, C);
    if (gl_better(e, k, be, bi)) { be = e; bi = k; }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float e2 = __shfl_xor_sync(0xffffffffu, be, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (gl_better(e2, i2, be, bi)) { be = e2; bi = i2; }
  }
  if (lane == 0) { s_e[warp] = be; s_i[warp] = bi; }
  __syncthreads();
  if (tid == 0) {
    for (int q = 1; q < NW; ++q)
      if (gl_better(s_e[q], s_i[q], be, bi)) { be = s_e[q]; bi = s_i[q]; }
    float C[9];
    if (bi >= 0) {
      float S[9];
#pragma unroll
      for (int q = 0; q < 9; ++q) S[q] = table[(size_t)(k0 + bi) * 9 + q];
      gl_matmul3(G, S, C);
    } else {
#pragma unroll
      for (int q = 0; q < 9; ++q) C[q] = G[q];
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) {
      s_rot[q] = C[q];
      w.rot_sel[(size_t)b * 9 + q] = C[q];
    }
    w.sym_idx[b] = bi;
    w.sym_err[b] = be;
  }
  __syncthreads();
  float Rs[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) Rs[q] = s_rot[q];
  float wt = 1.f;
  if (a.flags & F_PM_EXTENT) {
    const float* ex = gl_in<float>(a, IN_EXTENTS) + (size_t)b * 3;
    wt = __fdiv_rn(1.f, fmaxf(fmaxf(ex[0], ex[1]), ex[2]));
  }
  // sum |w R_est p - w R_gt' p| and sum sign(.) w p^T over the points
  double acc[10];
#pragma unroll
  for (int q = 0; q < 10; ++q) acc[q] = 0.0;
  const float* pts = gl_in<float>(a, IN_POINTS) + (size_t)b * a.N * 3;
  for (int n = tid; n < a.N; n += GL_PM_THREADS) {
    const float px = pts[3 * n], py = pts[3 * n + 1], pz = pts[3 * n + 2];
    const float wp[3] = {__fmul_rn(wt, px), __fmul_rn(wt, py), __fmul_rn(wt, pz)};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const float e = __fadd_rn(__fadd_rn(__fmul_rn(E[3 * i], px), __fmul_rn(E[3 * i + 1], py)), __fmul_rn(E[3 * i + 2], pz));
      const float g = __fadd_rn(__fadd_rn(__fmul_rn(Rs[3 * i], px), __fmul_rn(Rs[3 * i + 1], py)),
                                __fmul_rn(Rs[3 * i + 2], pz));
      const float d = __fsub_rn(__fmul_rn(wt, e), __fmul_rn(wt, g));
      acc[9] += fabsf(d);
      const float sg = gl_sign(d);
#pragma unroll
      for (int j = 0; j < 3; ++j) acc[3 * i + j] += __fmul_rn(sg, wp[j]);
    }
  }
#pragma unroll
  for (int q = 0; q < 10; ++q) {
    double v = acc[q];
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_acc[q][warp] = v;
  }
  __syncthreads();
  if (tid < 10) {
    double v = 0.0;
    for (int q = 0; q < NW; ++q) v += s_acc[tid][q];
    if (tid == 9) w.pm_abs[b] = v;
    else w.pm_sign[(size_t)b * 9 + tid] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------- stage 3
__global__ void __launch_bounds__(32) gl_finalize_kernel(GlArgs a, GlWs w) {
  __shared__ double s_sum[GL_NPART];
  const int tid = threadIdx.x, B = a.B, P = B * a.tiles;
  const bool geo = a.flags & F_GEO;
  if (tid < GL_NPART) {
    double v = 0.0;
    if (geo)
      for (int p = 0; p < P; ++p) v += w.partial[(size_t)p * GL_NPART + tid];
    s_sum[tid] = v;
  }
  __syncwarp();
  if (tid != 0) return;
  float* r = w.result;
  for (int q = 0; q < GL_NRES; ++q) r[q] = 0.f;
  const double n_xyz = fmax(s_sum[6], 1.0), n_reg = fmax(s_sum[7], 1.0), n_pix = (double)B * a.HW;
  const double n_pm = (double)B * a.N * 3;
  w.norm[0] = (float)n_xyz; w.norm[1] = (float)n_reg; w.norm[2] = (float)n_pix; w.norm[3] = (float)n_pm;
  int err = 0;
  if (geo) {
    for (int c = 0; c < 3; ++c) r[R_X + c] = (float)(s_sum[c] / n_xyz * a.w[W_XYZ]);
    r[R_MASK] = (float)(s_sum[3] / n_pix * a.w[W_MASK]);
    if (a.flags & F_FULL) r[R_FULL] = (float)(s_sum[4] / n_pix * a.w[W_FULL]);
    r[R_REGION] = (float)(s_sum[5] / n_reg * a.w[W_REGION]);
    for (int p = 0; p < P; ++p) err |= w.partial_err[p];
  }
  if (a.flags & F_PM) {
    double v = 0.0;
    for (int b = 0; b < B; ++b) v += w.pm_abs[b];
    r[R_PM] = (float)(3.0 * a.w[W_PM] * (v / n_pm));
  }
  if (a.flags & F_CENTROID) {
    const float* oc = gl_in<float>(a, IN_OUT_CENTROID);
    const float* gr = gl_in<float>(a, IN_GT_RATIO);
    double v = 0.0;
    for (int b = 0; b < B; ++b)
      for (int c = 0; c < 2; ++c) v += fabsf(__fsub_rn(oc[2 * b + c], gr[3 * b + c]));
    r[R_CENTROID] = (float)(v / (2.0 * B) * a.w[W_CENTROID]);
  }
  if (a.flags & F_Z) {
    const float* oz = gl_in<float>(a, IN_OUT_TZ);
    const float* gz = gl_in<float>(a, (a.flags & F_Z_ABS) ? IN_GT_TRANS : IN_GT_RATIO);
    double v = 0.0;
    for (int b = 0; b < B; ++b) v += fabsf(__fsub_rn(oz[b], gz[3 * b + 2]));
    r[R_TZ] = (float)(v / B * a.w[W_Z]);
  }
  r[R_ERR] = (float)err;
}

// ---------------------------------------------------------------------------------------------------------- stage 4
// Upstream gradient u of a returned loss (already times its weight) -> the scale of its elementwise gradient:
// (u * weight) / normaliser, in fp32 as torch's chain gives it.
__device__ __forceinline__ float gl_scale(float u, float weight, float norm) { return __fdiv_rn(__fmul_rn(u, weight), norm); }

struct GlGrads {
  float* g[G_COUNT];
};

// Grid (tiles, B) when the geometry terms are on, else (1, 1).  Map gradients from the stored log-sum-exp; CTA (0, 0)
// also writes the rotation, centroid and z gradients.
template <bool VEC>
__global__ void __launch_bounds__(GL_THREADS)
gl_backward_kernel(GlArgs a, GlWs w, const float* __restrict__ up, GlGrads gr) {
  const int b = blockIdx.y, tid = threadIdx.x, HW = a.HW, B = a.B;
  if (blockIdx.x == 0 && b == 0) {
    if (a.flags & F_PM) {
      const float s = gl_scale(up[R_PM], __fmul_rn(3.f, a.w[W_PM]), w.norm[3]);
      for (int e = tid; e < B * 9; e += GL_THREADS) gr.g[G_ROT][e] = (float)((double)s * w.pm_sign[e]);
    }
    if (a.flags & F_CENTROID) {
      const float s = gl_scale(up[R_CENTROID], a.w[W_CENTROID], (float)(2 * B));
      const float* oc = gl_in<float>(a, IN_OUT_CENTROID);
      const float* rt = gl_in<float>(a, IN_GT_RATIO);
      for (int e = tid; e < B * 2; e += GL_THREADS)
        gr.g[G_CENTROID][e] = __fmul_rn(gl_sign(__fsub_rn(oc[e], rt[3 * (e >> 1) + (e & 1)])), s);
    }
    if (a.flags & F_Z) {
      const float s = gl_scale(up[R_TZ], a.w[W_Z], (float)B);
      const float* oz = gl_in<float>(a, IN_OUT_TZ);
      const float* gz = gl_in<float>(a, (a.flags & F_Z_ABS) ? IN_GT_TRANS : IN_GT_RATIO);
      for (int e = tid; e < B; e += GL_THREADS) gr.g[G_TZ][e] = __fmul_rn(gl_sign(__fsub_rn(oz[e], gz[3 * e + 2])), s);
    }
  }
  if (!(a.flags & F_GEO)) return;
  const int p = blockIdx.x * GL_TILE + tid * GL_VEC;
  if (p >= HW) return;
  const size_t bp = (size_t)b * HW;
  float m[GL_VEC], o[GL_VEC], g[GL_VEC], d[GL_VEC];
  gl_ld<VEC>(gl_in<float>(a, IN_M_XYZ) + bp, p, HW, m);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float s = gl_scale(up[R_X + c], a.w[W_XYZ], w.norm[0]);
    gl_ld<VEC>(gl_in<float>(a, IN_OUT_X + c) + b * a.bs[c], p, HW, o);
    gl_ld<VEC>(gl_in<float>(a, IN_GT_XYZ) + (size_t)(3 * b + c) * HW, p, HW, g);
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j)
      d[j] = __fmul_rn(__fmul_rn(gl_sign(__fsub_rn(__fmul_rn(o[j], m[j]), __fmul_rn(g[j], m[j]))), s), m[j]);
    gl_st<VEC>(gr.g[G_X + c] + bp, p, HW, d);
  }
#pragma unroll
  for (int f = 0; f < 2; ++f) {
    if (f == 1 && !(a.flags & F_FULL)) break;
    const bool bce = a.flags & (f ? F_FULL_BCE : F_MASK_BCE);
    const float s = gl_scale(up[R_MASK + f], a.w[W_MASK + f], w.norm[2]);
    gl_ld<VEC>(gl_in<float>(a, f ? IN_OUT_FULL : IN_OUT_MASK) + b * a.bs[3 + f], p, HW, o);
    gl_ld<VEC>(gl_in<float>(a, f ? IN_M_FULL : IN_M_MASK) + bp, p, HW, m);
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j)
      d[j] = __fmul_rn(bce ? __fsub_rn(gl_sigmoid(o[j]), m[j]) : gl_sign(__fsub_rn(o[j], m[j])), s);
    gl_st<VEC>(gr.g[G_MASK + f] + bp, p, HW, d);
  }
  // region: ((exp(x - lse) - onehot) * s) * m with x = out m
  gl_ld<VEC>(gl_in<float>(a, IN_M_REGION) + bp, p, HW, m);
  const float s = gl_scale(up[R_REGION], a.w[W_REGION], w.norm[1]);
  const long long* lab = gl_in<long long>(a, IN_GT_REGION) + bp;
  float lse[GL_VEC];
  int t[GL_VEC];
  gl_ld<VEC>(w.lse + bp, p, HW, lse);
#pragma unroll
  for (int j = 0; j < GL_VEC; ++j) t[j] = p + j < HW ? (int)(lab[p + j] * (long long)m[j]) : 0;
  const float* reg = gl_in<float>(a, IN_OUT_REGION) + (size_t)b * a.R1 * HW;
  float* greg = gr.g[G_REGION] + (size_t)b * a.R1 * HW;
#pragma unroll 4
  for (int c = 0; c < a.R1; ++c) {
    gl_ld<VEC>(reg + (size_t)c * HW, p, HW, o);
#pragma unroll
    for (int j = 0; j < GL_VEC; ++j) {
      const float q = expf(__fsub_rn(__fmul_rn(o[j], m[j]), lse[j]));
      d[j] = __fmul_rn(__fmul_rn(c == t[j] ? __fsub_rn(q, 1.f) : q, s), m[j]);
    }
    gl_st<VEC>(greg + (size_t)c * HW, p, HW, d);
  }
}

// the float4 path needs every plane it touches 16-byte aligned: base pointers, batch strides and HW
bool gl_vec_ok(const GlArgs& a) {
  if (a.HW % 4) return false;
  for (int k = 0; k < IN_COUNT; ++k)
    if (a.in[k] && (reinterpret_cast<uintptr_t>(a.in[k]) & 15)) return false;
  for (int k = 0; k < 5; ++k)
    if (a.bs[k] % 4) return false;
  return true;
}

}  // namespace

extern "C" size_t gdrn_loss_workspace_bytes(int B, int HW) {
  if (B <= 0 || HW <= 0) return 0;
  return gl_layout(B, HW).off[GL_NOFF] + 256;
}

extern "C" int gdrn_loss_layout(int B, int HW, size_t* offsets) {
  GDRN_REQUIRE(offsets && B > 0 && HW > 0, "gdrn_loss_layout: bad arguments");
  const GlLayout l = gl_layout(B, HW);
  for (int k = 0; k < GL_NOFF; ++k) offsets[k] = l.off[k];
  return GDRN_OK;
}

static int gl_args(const void* const* inputs, const long long* batch_strides, const float* weights, int B, int HW, int R1,
                   int N, int flags, void* workspace, size_t workspace_bytes, GlArgs* a) {
  GDRN_REQUIRE(inputs && batch_strides && weights && workspace, "gdrn_loss: null argument");
  GDRN_REQUIRE(B > 0 && HW > 0 && R1 > 0 && N >= 0, "gdrn_loss: empty problem");
  GDRN_REQUIRE(workspace_bytes >= gdrn_loss_workspace_bytes(B, HW), "gdrn_loss: workspace too small");
  for (int k = 0; k < IN_COUNT; ++k) a->in[k] = inputs[k];
  for (int k = 0; k < 5; ++k) a->bs[k] = batch_strides[k];
  for (int k = 0; k < W_COUNT; ++k) a->w[k] = weights[k];
  a->B = B; a->HW = HW; a->R1 = R1; a->N = N; a->flags = flags; a->tiles = gl_tiles(HW);
  if (flags & F_GEO) {
    GDRN_REQUIRE(a->in[IN_OUT_X] && a->in[IN_OUT_Y] && a->in[IN_OUT_Z] && a->in[IN_OUT_MASK] && a->in[IN_M_XYZ] &&
                 a->in[IN_M_MASK] && a->in[IN_M_REGION] && a->in[IN_GT_XYZ] && a->in[IN_OUT_REGION] &&
                 a->in[IN_GT_REGION], "gdrn_loss: a geometry input is null");
    GDRN_REQUIRE(!(flags & F_FULL) || (a->in[IN_OUT_FULL] && a->in[IN_M_FULL]), "gdrn_loss: a full-mask input is null");
  }
  GDRN_REQUIRE(!(flags & F_PM) || (a->in[IN_OUT_ROT] && a->in[IN_GT_ROT] && a->in[IN_POINTS] && N > 0),
               "gdrn_loss: point matching needs out_rot, gt_rot and points");
  GDRN_REQUIRE(!(flags & F_PM_EXTENT) || a->in[IN_EXTENTS], "gdrn_loss: PM_NORM_BY_EXTENT needs extents");
  GDRN_REQUIRE(!a->in[IN_SYM_RANGE] || a->in[IN_SYM_TABLE], "gdrn_loss: symmetry ranges without a table");
  GDRN_REQUIRE(!(flags & F_CENTROID) || (a->in[IN_OUT_CENTROID] && a->in[IN_GT_RATIO]),
               "gdrn_loss: the centroid term needs out_centroid and gt_trans_ratio");
  GDRN_REQUIRE(!(flags & F_Z) || (a->in[IN_OUT_TZ] && a->in[(flags & F_Z_ABS) ? IN_GT_TRANS : IN_GT_RATIO]),
               "gdrn_loss: the z term needs out_trans_z and its target");
  return GDRN_OK;
}

extern "C" int gdrn_loss_forward(const void* const* inputs, const long long* batch_strides, const float* weights, int B,
                                 int HW, int R1, int N, int flags, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  GlArgs a;
  const int rc = gl_args(inputs, batch_strides, weights, B, HW, R1, N, flags, workspace, workspace_bytes, &a);
  if (rc != GDRN_OK) return rc;
  const GlWs w = gl_ws(workspace, B, HW);
  cudaStream_t st = (cudaStream_t)stream;
  int n = 1;
  if (flags & F_GEO) {
    if (gl_vec_ok(a)) gl_dense_kernel<true><<<dim3(a.tiles, B), GL_THREADS, 0, st>>>(a, w);
    else gl_dense_kernel<false><<<dim3(a.tiles, B), GL_THREADS, 0, st>>>(a, w);
    ++n;
  }
  if (flags & F_PM) {
    gl_pm_kernel<<<B, GL_PM_THREADS, 0, st>>>(a, w);
    ++n;
  }
  gl_finalize_kernel<<<1, 32, 0, st>>>(a, w);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(n);
  return GDRN_OK;
}

extern "C" int gdrn_loss_backward(const void* const* inputs, const long long* batch_strides, const float* weights,
                                  int B, int HW, int R1, int N, int flags, const float* grad_losses,
                                  void* const* grads, void* workspace, size_t workspace_bytes, void* stream) {
  GlArgs a;
  const int rc = gl_args(inputs, batch_strides, weights, B, HW, R1, N, flags, workspace, workspace_bytes, &a);
  if (rc != GDRN_OK) return rc;
  GDRN_REQUIRE(grad_losses && grads, "gdrn_loss_backward: null gradient argument");
  GlGrads gr;
  for (int k = 0; k < G_COUNT; ++k) gr.g[k] = static_cast<float*>(grads[k]);
  GDRN_REQUIRE(!(flags & F_GEO) || (gr.g[G_X] && gr.g[G_Y] && gr.g[G_Z] && gr.g[G_MASK] && gr.g[G_REGION] &&
                                    (!(flags & F_FULL) || gr.g[G_FULL])), "gdrn_loss_backward: a map gradient is null");
  GDRN_REQUIRE(!(flags & F_PM) || gr.g[G_ROT], "gdrn_loss_backward: the rotation gradient is null");
  GDRN_REQUIRE(!(flags & F_CENTROID) || gr.g[G_CENTROID], "gdrn_loss_backward: the centroid gradient is null");
  GDRN_REQUIRE(!(flags & F_Z) || gr.g[G_TZ], "gdrn_loss_backward: the z gradient is null");
  const GlWs w = gl_ws(workspace, B, HW);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid = (flags & F_GEO) ? dim3(a.tiles, B) : dim3(1, 1);
  bool vec = (flags & F_GEO) && gl_vec_ok(a);
  for (int k = 0; k < 6 && vec; ++k) vec = !gr.g[k] || !(reinterpret_cast<uintptr_t>(gr.g[k]) & 15);
  if (vec) gl_backward_kernel<true><<<grid, GL_THREADS, 0, st>>>(a, w, grad_losses, gr);
  else gl_backward_kernel<false><<<grid, GL_THREADS, 0, st>>>(a, w, grad_losses, gr);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
