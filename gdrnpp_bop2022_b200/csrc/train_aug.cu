// The training image pipeline of the reference's GDRN_Online_DatasetFromList.read_data_train
// (core/gdrn_modeling/datasets/data_loader_online.py:311-581) for a whole batch of uint8 BGR images [n,H,W,3]:
//   gdrn_train_composite   background replacement (base_data_loader.py replace_bg / trunc_mask / get_bg_image): the
//                          visible mask's bounding box reduced on the device, the truncation window cut from it, the
//                          background's top-left crop resized with cv2's bilinear arithmetic (cv_resize.cuh) and pasted
//                          where the (truncated) mask is off;
//   gdrn_train_luma_sum    PIL's L-image sum of the images whose colour op at one step is EnhanceContrast;
//   gdrn_train_color_step  one position of imgaug's random_order Sequential: image b gets op kind_at[b][step] (or passes
//                          through), uint8 in, uint8 out, ping-pong buffers;
//   gdrn_train_roi_crop    the DZI-jittered crops (crop_common.cuh, bit-exact cv2.warpAffine): roi_img, roi_coord_2d and
//                          the nearest-neighbour trunc / visib / full masks, with each ROI's trunc and visib pixel counts.
// Every random choice arrives from the host in the per-sample record (gdrnpp_bop2022_b200/train_batch.py); the kernels
// are deterministic functions of (images, record).  No FMA contraction anywhere: explicit _rn intrinsics.
#include "crop_common.cuh"
#include "cv_resize.cuh"

namespace {

// colour-op kinds; the host (train_batch.py COLOR_OPS) uses the same numbering
enum ColorOp {
  kDropout = 0, kBlur = 1, kSharpness = 2, kContrast = 3, kBrightness = 4, kColor = 5, kAdd = 6, kInvert = 7,
  kMultiply = 8, kNoise = 9, kLinearContrast = 10, kGrayscale = 11
};
constexpr int kFPar = 4, kIPar = 12;

__device__ __forceinline__ int clip255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// PIL's ITU-R 601-2 L conversion (channel 0 taken as R, as PIL sees a BGR array)
__device__ __forceinline__ int pil_luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// cv2.cvtColor(COLOR_RGB2GRAY) on uint8 as its vectorised path computes it: 15-bit fixed point
__device__ __forceinline__ int cv_gray(int r, int g, int b) { return (r * 9798 + g * 19235 + b * 3735 + (1 << 14)) >> 15; }

// PIL ImagingBlend(degenerate, image, alpha): float arithmetic, truncation, clipped when extrapolating
__device__ __forceinline__ int pil_blend(int deg, int im, float a) {
  const float t = __fadd_rn((float)deg, __fmul_rn(a, (float)(im - deg)));
  if (t <= 0.f) return 0;
  if (t >= 255.f) return 255;
  return (int)t;
}

__device__ __forceinline__ int rint_clip(double v) { return clip255(__double2int_rn(v)); }

__device__ __forceinline__ int reflect101(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

// Philox4x32-10 (Salmon et al., SC'11): counter (c0, 0, 0, 0), key (k0, k1)
__device__ __forceinline__ void philox4x32(unsigned c0, unsigned k0, unsigned k1, unsigned (&r)[4]) {
  unsigned x0 = c0, x1 = 0, x2 = 0, x3 = 0;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const unsigned long long p0 = 0xD2511F53ull * x0, p1 = 0xCD9E8D57ull * x2;
    const unsigned y0 = (unsigned)(p1 >> 32) ^ x1 ^ k0, y2 = (unsigned)(p0 >> 32) ^ x3 ^ k1;
    x1 = (unsigned)p1;
    x3 = (unsigned)p0;
    x0 = y0;
    x2 = y2;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  r[0] = x0; r[1] = x1; r[2] = x2; r[3] = x3;
}

// uniform in (0, 1]: (r + 1) / 2^32
__device__ __forceinline__ double u01(unsigned r) { return __dmul_rn((double)r + 1.0, 2.3283064365386963e-10); }

// ---------------------------------------------------------------------------------------------------- background
__global__ void __launch_bounds__(256)
mask_bbox_kernel(const uint8_t* __restrict__ mask, int H, int W, int* __restrict__ bbox) {
  const int b = blockIdx.y;
  const long long plane = (long long)H * W;
  int rmin = H, rmax = -1, cmin = W, cmax = -1;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < plane; p += (long long)gridDim.x * blockDim.x) {
    if (mask[b * plane + p]) {
      const int y = (int)(p / W), x = (int)(p % W);
      rmin = min(rmin, y); rmax = max(rmax, y); cmin = min(cmin, x); cmax = max(cmax, x);
    }
  }
  rmin = __reduce_min_sync(0xffffffffu, rmin);
  rmax = __reduce_max_sync(0xffffffffu, rmax);
  cmin = __reduce_min_sync(0xffffffffu, cmin);
  cmax = __reduce_max_sync(0xffffffffu, cmax);
  if ((threadIdx.x & 31) == 0 && rmax >= 0) {
    atomicMin(bbox + 4 * b, rmin); atomicMax(bbox + 4 * b + 1, rmax);
    atomicMin(bbox + 4 * b + 2, cmin); atomicMax(bbox + 4 * b + 3, cmax);
  }
}

// trunc_mask (base_data_loader.py:454-478): c = int(random.uniform(a, b)) = int(a + (b - a) * u); side 0 clears the rows
// above c, 1 the rows from c, 2 the columns left of c, 3 the columns from c; any other side keeps the whole mask.
// keep = [row0, row1, col0, col1) of the window the truncated mask keeps.
__global__ void trunc_window_kernel(const int* __restrict__ bbox, const int* __restrict__ side, const double* __restrict__ u,
                                    int n, int H, int W, int* __restrict__ keep) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  int k[4] = {0, H, 0, W};
  const int s = side[b];
  if (s >= 0 && s < 4) {
    const double lo = s < 2 ? bbox[4 * b] : bbox[4 * b + 2], hi = s < 2 ? bbox[4 * b + 1] : bbox[4 * b + 3];
    const double c = __dmul_rn(0.5, __dadd_rn(lo, hi));
    const double a = (s & 1) ? c : lo, e = (s & 1) ? hi : c;
    const int cut = (int)__dadd_rn(a, __dmul_rn(__dsub_rn(e, a), u[b]));
    if (s == 0) k[0] = cut; else if (s == 1) k[1] = cut; else if (s == 2) k[2] = cut; else k[3] = cut;
  }
  for (int i = 0; i < 4; ++i) keep[4 * b + i] = k[i];
}

// bg_meta per sample: do_bg, bg_h, bg_w, crop_h, crop_w, resized_h, resized_w; bg_scale: (1 / fx, 1 / fy)
__global__ void __launch_bounds__(256)
composite_kernel(uint8_t* __restrict__ images, const uint8_t* __restrict__ mask, int n, int H, int W,
                 const uint8_t* __restrict__ bg_pool, const long long* __restrict__ bg_off, const int* __restrict__ bg_meta,
                 const double* __restrict__ bg_scale, const int* __restrict__ keep) {
  const long long plane = (long long)H * W;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= plane * n) return;
  const int b = (int)(idx / plane);
  const int* m = bg_meta + 7 * b;
  if (!m[0]) return;
  const int y = (int)((idx % plane) / W), x = (int)(idx % W);
  const int* k = keep + 4 * b;
  if (mask[idx] && y >= k[0] && y < k[1] && x >= k[2] && x < k[3]) return;
  int v[3] = {0, 0, 0};
  if (y < m[5] && x < m[6]) {
    const int mode = cvresize::resize_mode(m[3], m[4], m[5], m[6], bg_scale[2 * b], bg_scale[2 * b + 1]);
    cvresize::pixel_u8(bg_pool + bg_off[b], 3LL * m[2], m[3], m[4], 3, x, y, mode, bg_scale[2 * b], bg_scale[2 * b + 1], v);
  }
  uint8_t* o = images + idx * 3;
  o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
}

// ---------------------------------------------------------------------------------------------------- colour
__global__ void __launch_bounds__(256)
luma_sum_kernel(const uint8_t* __restrict__ img, int H, int W, const int* __restrict__ kind_at, int S, int step,
                unsigned long long* __restrict__ sums) {
  const int b = blockIdx.y;
  if (kind_at[b * S + step] != kContrast) return;
  const long long plane = (long long)H * W;
  unsigned s = 0;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < plane; p += (long long)gridDim.x * blockDim.x) {
    const uint8_t* q = img + (b * plane + p) * 3;
    s += pil_luma(q[0], q[1], q[2]);
  }
  s = __reduce_add_sync(0xffffffffu, s);
  if ((threadIdx.x & 31) == 0) atomicAdd(sums + b, (unsigned long long)s);
}

__global__ void __launch_bounds__(256)
color_step_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int n, int H, int W,
                  const int* __restrict__ kind_at, const float* __restrict__ fpar, const int* __restrict__ ipar, int S,
                  int step, const uint8_t* __restrict__ cells, int ch, int cw, const unsigned long long* __restrict__ luma_sums) {
  const long long plane = (long long)H * W;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= plane * n) return;
  const int b = (int)(idx / plane);
  const int y = (int)((idx % plane) / W), x = (int)(idx % W);
  const uint8_t* img = src + b * plane * 3;
  const uint8_t* p = src + idx * 3;
  const int kind = kind_at[b * S + step];
  const float* fp = fpar + (long long)(b * S + step) * kFPar;
  const int* ip = ipar + (long long)(b * S + step) * kIPar;
  int v[3] = {p[0], p[1], p[2]};
  switch (kind) {
    case kDropout: {   // the cell grid nearest-upsampled as cv2.resize(INTER_NEAREST): floor(x * (1 / (W / cw)))
      const int sy = min((int)floor(__dmul_rn((double)y, 1.0 / ((double)H / ch))), ch - 1);
      const int sx = min((int)floor(__dmul_rn((double)x, 1.0 / ((double)W / cw))), cw - 1);
      if (!cells[(long long)b * ch * cw + sy * cw + sx]) v[0] = v[1] = v[2] = 0;
      break;
    }
    case kBlur: {   // cv2.GaussianBlur's fixed-point 8-bit path: 8-bit coefficients, 16-bit rounding shift
      const int K = ip[0], r = K / 2;
      int acc[3] = {0, 0, 0};
      for (int i = 0; i < K; ++i) {
        const uint8_t* row = img + (long long)reflect101(y + i - r, H) * W * 3;
        int h[3] = {0, 0, 0};
        for (int j = 0; j < K; ++j) {
          const uint8_t* q = row + reflect101(x + j - r, W) * 3;
          h[0] += ip[1 + j] * q[0]; h[1] += ip[1 + j] * q[1]; h[2] += ip[1 + j] * q[2];
        }
        acc[0] += ip[1 + i] * h[0]; acc[1] += ip[1 + i] * h[1]; acc[2] += ip[1 + i] * h[2];
      }
      for (int c = 0; c < 3; ++c) v[c] = clip255((acc[c] + 32768) >> 16);
      break;
    }
    case kSharpness: {   // PIL ImageFilter.SMOOTH (3x3 [1 1 1; 1 5 1; 1 1 1] / 13, border copied), then blend
      if (y > 0 && y < H - 1 && x > 0 && x < W - 1) {
        const float k1 = __fdiv_rn(1.f, 13.f), k5 = __fdiv_rn(5.f, 13.f);
        for (int c = 0; c < 3; ++c) {
          float ss = 0.f;
          for (int dy = -1; dy <= 1; ++dy) {
            const uint8_t* q = p + (long long)dy * W * 3;
            const float kc = dy == 0 ? k5 : k1;
            ss = __fadd_rn(ss, __fadd_rn(__fadd_rn(__fmul_rn((float)q[c - 3], k1), __fmul_rn((float)q[c], kc)),
                                         __fmul_rn((float)q[c + 3], k1)));
          }
          ss = __fadd_rn(ss, 0.5f);
          const int deg = ss <= 0.f ? 0 : (ss >= 255.f ? 255 : (int)ss);
          v[c] = pil_blend(deg, v[c], fp[0]);
        }
      }
      break;
    }
    case kContrast: {   // degenerate = int(mean(L) + 0.5) everywhere
      const double mean = __ddiv_rn((double)luma_sums[b], (double)plane);
      const int m = (int)floor(__dadd_rn(mean, 0.5));
      for (int c = 0; c < 3; ++c) v[c] = pil_blend(m, v[c], fp[0]);
      break;
    }
    case kBrightness:
      for (int c = 0; c < 3; ++c) v[c] = pil_blend(0, v[c], fp[0]);
      break;
    case kColor: {
      const int l = pil_luma(v[0], v[1], v[2]);
      for (int c = 0; c < 3; ++c) v[c] = pil_blend(l, v[c], fp[0]);
      break;
    }
    case kAdd:
      for (int c = 0; c < 3; ++c) v[c] = clip255(v[c] + ip[c]);
      break;
    case kInvert:
      for (int c = 0; c < 3; ++c) if (ip[c]) v[c] = 255 - v[c];
      break;
    case kMultiply:
      for (int c = 0; c < 3; ++c) v[c] = rint_clip(__dmul_rn((double)v[c], (double)fp[c]));
      break;
    case kNoise: {   // N(0, scale) per channel: Box-Muller on Philox4x32-10 of (pixel index; seed)
      unsigned r[4];
      philox4x32((unsigned)(idx % plane), (unsigned)ip[0], (unsigned)ip[1], r);
      const double twopi = 6.283185307179586;
      const double ra = sqrt(__dmul_rn(-2.0, log(u01(r[0])))), rb = sqrt(__dmul_rn(-2.0, log(u01(r[2]))));
      const double ta = __dmul_rn(twopi, u01(r[1])), tb = __dmul_rn(twopi, u01(r[3]));
      const double z[3] = {__dmul_rn(ra, cos(ta)), __dmul_rn(ra, sin(ta)), __dmul_rn(rb, cos(tb))};
      for (int c = 0; c < 3; ++c) v[c] = rint_clip(__dadd_rn((double)v[c], __dmul_rn((double)fp[0], z[c])));
      break;
    }
    case kLinearContrast:   // 127.5 + alpha (v - 127.5)
      for (int c = 0; c < 3; ++c) v[c] = rint_clip(__dadd_rn(127.5, __dmul_rn((double)fp[c], __dsub_rn((double)v[c], 127.5))));
      break;
    case kGrayscale: {   // alpha-blend towards cv2's RGB2GRAY luma
      const double a = fp[0], g = cv_gray(v[0], v[1], v[2]);
      for (int c = 0; c < 3; ++c) v[c] = rint_clip(__dadd_rn(__dmul_rn(g, a), __dmul_rn((double)v[c], __dsub_rn(1.0, a))));
      break;
    }
    default:
      break;
  }
  uint8_t* o = dst + idx * 3;
  o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
}

// ---------------------------------------------------------------------------------------------------- ROI crops
// Blocks [0, n_big) cover roi_img (in_res), the rest the out_res outputs.  One thread per output pixel of one ROI.
__global__ void __launch_bounds__(256)
train_crop_kernel(const uint8_t* __restrict__ images, const uint8_t* __restrict__ mvis, const uint8_t* __restrict__ mfull,
                  const int* __restrict__ keep, const double* __restrict__ cs, int n, int H, int W, int in_res, int out_res,
                  long long n_big, double m0, double m1, double m2, double s0, double s1, double s2,
                  float* __restrict__ roi_img, float* __restrict__ roi_coord_2d, float* __restrict__ roi_trunc,
                  float* __restrict__ roi_visib, float* __restrict__ roi_full, int* __restrict__ counts) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long plane = (long long)H * W;
  if (idx < n_big) {
    const long long per = (long long)in_res * in_res;
    if (idx >= per * n) return;
    const int b = (int)(idx / per);
    const int y = (int)((idx % per) / in_res), x = (int)(idx % in_res);
    double iM[6];
    crop::invert_affine(crop::forward_affine(cs[3 * b], cs[3 * b + 1], cs[3 * b + 2], in_res).m, iM);
    const crop::U8Tap t = crop::u8_tap(crop::src_coord(iM, x, y, false), H, W);
    const uint8_t* p00 = images + (b * plane + (long long)t.sy * W + t.sx) * 3;
    const long long rowC = (long long)W * 3;
    const double mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
    const long long o = (long long)b * 3 * per + (long long)y * in_res + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int v = 0;
      if (t.in[0]) v += p00[c] * t.w[0];
      if (t.in[1]) v += p00[3 + c] * t.w[1];
      if (t.in[2]) v += p00[rowC + c] * t.w[2];
      if (t.in[3]) v += p00[rowC + 3 + c] * t.w[3];
      v = crop::u8_round(v);
      roi_img[o + c * per] = __double2float_rn(__ddiv_rn(__dsub_rn((double)v, mean[c]), stdv[c]));
    }
    return;
  }
  const long long j = idx - n_big;
  const long long per = (long long)out_res * out_res;
  bool tr = false, vi = false;
  if (j < per * n) {
    const int b = (int)(j / per);
    const int y = (int)((j % per) / out_res), x = (int)(j % out_res);
    double iM[6];
    crop::invert_affine(crop::forward_affine(cs[3 * b], cs[3 * b + 1], cs[3 * b + 2], out_res).m, iM);
    const crop::F32Tap t = crop::f32_tap(crop::src_coord(iM, x, y, false), H, W);
    const float gx0 = crop::grid_value(t.sx, W), gx1 = crop::grid_value(t.sx + 1, W);
    const float gy0 = crop::grid_value(t.sy, H), gy1 = crop::grid_value(t.sy + 1, H);
    const long long o = (long long)b * 2 * per + (long long)y * out_res + x;
    roi_coord_2d[o] = crop::f32_blend(t, t.in[0] ? gx0 : 0.f, t.in[1] ? gx1 : 0.f, t.in[2] ? gx0 : 0.f, t.in[3] ? gx1 : 0.f);
    roi_coord_2d[o + per] = crop::f32_blend(t, t.in[0] ? gy0 : 0.f, t.in[1] ? gy0 : 0.f, t.in[2] ? gy1 : 0.f, t.in[3] ? gy1 : 0.f);
    const crop::SrcCoord sc = crop::src_coord(iM, x, y, true);
    bool fu = false;
    if (sc.X >= 0 && sc.X < W && sc.Y >= 0 && sc.Y < H) {
      const long long q = b * plane + (long long)sc.Y * W + sc.X;
      const int* k = keep + 4 * b;
      vi = mvis[q] != 0;
      fu = mfull[q] != 0;
      tr = vi && sc.Y >= k[0] && sc.Y < k[1] && sc.X >= k[2] && sc.X < k[3];
    }
    const long long om = (long long)b * per + (long long)y * out_res + x;
    roi_trunc[om] = tr ? 1.f : 0.f;
    roi_visib[om] = vi ? 1.f : 0.f;
    roi_full[om] = fu ? 1.f : 0.f;
  }
  // per-ROI pixel counts; a warp may straddle two ROIs, so split the ballot by ROI
  const int b = j < per * n ? (int)(j / per) : -1;
  const unsigned act = __activemask();
  const unsigned same = __match_any_sync(act, b);
  const int ct = __popc(__ballot_sync(act, tr) & same), cv = __popc(__ballot_sync(act, vi) & same);
  if (b >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) {
    if (ct) atomicAdd(counts + 2 * b, ct);
    if (cv) atomicAdd(counts + 2 * b + 1, cv);
  }
}

}  // namespace

extern "C" int gdrn_train_composite(uint8_t* images, const uint8_t* mask_visib, int n, int H, int W, const uint8_t* bg_pool,
                                    const long long* bg_off, const int* bg_meta, const double* bg_scale, const int* side,
                                    const double* trunc_u, int* bbox, int* keep, void* stream) {
  GDRN_REQUIRE(n >= 0 && H > 0 && W > 0, "train_composite: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(images && mask_visib && bg_off && bg_meta && bg_scale && side && trunc_u && bbox && keep,
               "train_composite: null argument");
  const cudaStream_t s = (cudaStream_t)stream;
  // bbox starts as (H, -1, W, -1) per sample: written by the host
  const long long plane = (long long)H * W;
  const int bx = (int)min((plane + 255) / 256, 64LL);
  mask_bbox_kernel<<<dim3(bx, n), 256, 0, s>>>(mask_visib, H, W, bbox);
  GDRN_CHECK_CUDA(cudaGetLastError());
  trunc_window_kernel<<<(n + 127) / 128, 128, 0, s>>>(bbox, side, trunc_u, n, H, W, keep);
  GDRN_CHECK_CUDA(cudaGetLastError());
  composite_kernel<<<(unsigned)((plane * n + 255) / 256), 256, 0, s>>>(images, mask_visib, n, H, W, bg_pool, bg_off, bg_meta,
                                                                      bg_scale, keep);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(3);
  return GDRN_OK;
}

extern "C" int gdrn_train_luma_sum(const uint8_t* images, int n, int H, int W, const int* kind_at, int S, int step,
                                   unsigned long long* sums, void* stream) {
  GDRN_REQUIRE(n >= 0 && H > 0 && W > 0 && S > 0 && step >= 0 && step < S, "train_luma_sum: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(images && kind_at && sums, "train_luma_sum: null argument");
  const cudaStream_t s = (cudaStream_t)stream;
  GDRN_CHECK_CUDA(cudaMemsetAsync(sums, 0, sizeof(unsigned long long) * n, s));
  const long long plane = (long long)H * W;
  luma_sum_kernel<<<dim3((unsigned)min((plane + 255) / 256, 64LL), n), 256, 0, s>>>(images, H, W, kind_at, S, step, sums);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_train_color_step(const uint8_t* src, uint8_t* dst, int n, int H, int W, const int* kind_at,
                                     const float* fpar, const int* ipar, int S, int step, const uint8_t* cells, int ch,
                                     int cw, const unsigned long long* luma_sums, void* stream) {
  GDRN_REQUIRE(n >= 0 && H > 0 && W > 0 && S > 0 && step >= 0 && step < S && ch > 0 && cw > 0, "train_color_step: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(src && dst && src != dst && kind_at && fpar && ipar && cells && luma_sums, "train_color_step: null argument");
  const long long total = (long long)n * H * W;
  color_step_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      src, dst, n, H, W, kind_at, fpar, ipar, S, step, cells, ch, cw, luma_sums);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_train_roi_crop(const uint8_t* images, const uint8_t* mask_visib, const uint8_t* mask_full,
                                   const int* keep, const double* center_scale, int n, int H, int W, int in_res, int out_res,
                                   const double* pixel_mean, const double* pixel_std, float* roi_img, float* roi_coord_2d,
                                   float* roi_mask_trunc, float* roi_mask_visib, float* roi_mask_full, int* counts,
                                   void* stream) {
  GDRN_REQUIRE(n >= 0 && H > 0 && W > 0 && in_res > 0 && out_res > 0, "train_roi_crop: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(images && mask_visib && mask_full && keep && center_scale && pixel_mean && pixel_std && roi_img &&
                   roi_coord_2d && roi_mask_trunc && roi_mask_visib && roi_mask_full && counts,
               "train_roi_crop: null argument");
  const cudaStream_t s = (cudaStream_t)stream;
  GDRN_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 2 * n, s));
  const long long big = (long long)n * in_res * in_res, small = (long long)n * out_res * out_res;
  const long long big_blocks = (big + 255) / 256, small_blocks = (small + 255) / 256;
  train_crop_kernel<<<(unsigned)(big_blocks + small_blocks), 256, 0, s>>>(
      images, mask_visib, mask_full, keep, center_scale, n, H, W, in_res, out_res, big_blocks * 256, pixel_mean[0],
      pixel_mean[1], pixel_mean[2], pixel_std[0], pixel_std[1], pixel_std[2], roi_img, roi_coord_2d, roi_mask_trunc,
      roi_mask_visib, roi_mask_full, counts);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
