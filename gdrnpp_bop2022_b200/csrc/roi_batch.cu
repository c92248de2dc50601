// Model inputs for the ROIs of many images at once: the per-ROI bookkeeping of the reference's test data loader
// (datasets/data_loader.py:751-797 read_data_test, then engine/engine_utils.py:213-241 batch_data_test) and every
// crop of the batch (image, 2-D coordinate grid, depth, depth-refine sensor crop) in one launch each.
//
// gdrn_roi_setup follows the reference's dtype path step for step (no FMA contraction anywhere):
//   bbox_est xywh -> BoxMode.convert through a float32 torch tensor: x2 = f32(x + w), y2 = f32(y + h);
//   centre = 0.5 * (x1 + x2), bw = max(x2 - x1, 1), scale = min(max(bh, bw) * DZI_PAD_SCALE, max(H, W)),
//   resize_ratio = out_res / scale, all in float64; batch_data_test rounds them to float32.
//   M = get_affine_transform(centre f64, (scale, scale) f64 -- crop_resize_by_warp_affine wraps the scale in a tuple,
//   so it stays float64 --, 0, res): the three float32 point pairs it builds are
//     src (X0, Y0), (X0, Y1), (X2, Y1) with X0 = f32(cx), Y0 = f32(cy), Y1 = f32(cy - scale / 2),
//     X2 = f32(X0 - f32(Y0 - Y1)), and dst (r/2, r/2), (r/2, 0), (0, 0);
//   their affine map is diagonal and solved here in closed form in float64.
// gdrn_roi_crop_multi reproduces crop_resize.cu's arithmetic (crop_common.cuh) with the source picked per ROI.
#include "crop_common.cuh"

namespace {

__global__ void __launch_bounds__(128)
roi_setup_kernel(const int* __restrict__ det_meta, const float* __restrict__ det_xywh, int n, const float* __restrict__ K,
                 const int* __restrict__ im_hw, const float* __restrict__ extents, double dzi_pad_scale, int in_res,
                 int out_res, float* __restrict__ roi_center, float* __restrict__ roi_wh, float* __restrict__ scale_out,
                 float* __restrict__ resize_ratio, float* __restrict__ roi_extent, float* __restrict__ roi_cam,
                 long long* __restrict__ roi_cls, float* __restrict__ im_H_out, float* __restrict__ im_W_out,
                 float* __restrict__ bbox_xyxy, double* __restrict__ M_in, double* __restrict__ M_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int img = det_meta[2 * i], label = det_meta[2 * i + 1];
  const float x = det_xywh[4 * i], y = det_xywh[4 * i + 1];
  const float x2f = __fadd_rn(x, det_xywh[4 * i + 2]), y2f = __fadd_rn(y, det_xywh[4 * i + 3]);
  const double x1 = x, y1 = y, x2 = x2f, y2 = y2f;
  const double cx = __dmul_rn(0.5, __dadd_rn(x1, x2)), cy = __dmul_rn(0.5, __dadd_rn(y1, y2));
  double bw = __dsub_rn(x2, x1), bh = __dsub_rn(y2, y1);
  bw = bw < 1.0 ? 1.0 : bw;
  bh = bh < 1.0 ? 1.0 : bh;
  const int H = im_hw[2 * img], W = im_hw[2 * img + 1];
  double scale = __dmul_rn(bw > bh ? bw : bh, dzi_pad_scale);
  const double max_hw = (double)(H > W ? H : W);
  scale = max_hw < scale ? max_hw : scale;
  roi_center[2 * i] = __double2float_rn(cx);
  roi_center[2 * i + 1] = __double2float_rn(cy);
  roi_wh[2 * i] = __double2float_rn(bw);
  roi_wh[2 * i + 1] = __double2float_rn(bh);
  scale_out[i] = __double2float_rn(scale);
  resize_ratio[i] = __double2float_rn(__ddiv_rn((double)out_res, scale));
  for (int k = 0; k < 3; ++k) roi_extent[3 * i + k] = extents[3 * label + k];
  for (int k = 0; k < 9; ++k) roi_cam[9 * i + k] = K[9 * img + k];
  roi_cls[i] = label;
  im_H_out[i] = (float)H;
  im_W_out[i] = (float)W;
  bbox_xyxy[4 * i] = x; bbox_xyxy[4 * i + 1] = y; bbox_xyxy[4 * i + 2] = x2f; bbox_xyxy[4 * i + 3] = y2f;
  const crop::Affine6 a_in = crop::forward_affine(cx, cy, scale, in_res), a_out = crop::forward_affine(cx, cy, scale, out_res);
  for (int k = 0; k < 6; ++k) { M_in[6 * i + k] = a_in.m[k]; M_out[6 * i + k] = a_out.m[k]; }
}

// metres as mmcv.imread(depth) / depth_factor, then astype(float32)
__device__ __forceinline__ float depth_m(const uint16_t* __restrict__ d, int W, int sx, int sy, double factor) {
  return __double2float_rn(__ddiv_rn((double)d[(long long)sy * W + sx], factor));
}

__device__ __forceinline__ float depth_nearest(const uint16_t* __restrict__ d, int H, int W, const double (&iM)[6], int x, int y,
                                               double factor) {
  const crop::SrcCoord sc = crop::src_coord(iM, x, y, true);
  return (sc.X >= 0 && sc.X < W && sc.Y >= 0 && sc.Y < H) ? depth_m(d, W, sc.X, sc.Y, factor) : 0.f;
}

// Blocks [0, n_big) cover the in_res x in_res outputs (roi_img, roi_depth), the rest the out_res x out_res ones
// (roi_coord_2d, the depth-refine sensor crop).  One thread per output pixel of one ROI.
__global__ void __launch_bounds__(256)
roi_crop_multi_kernel(const uint8_t* __restrict__ images, int H, int W, int C, const int* __restrict__ det_meta,
                      const double* __restrict__ M_in, const double* __restrict__ M_out, int n, int in_res, int out_res,
                      long long n_big, double m0, double m1, double m2, double s0, double s1, double s2,
                      const uint16_t* __restrict__ depth, const double* __restrict__ depth_factor,
                      float* __restrict__ roi_img, float* __restrict__ roi_coord_2d, float* __restrict__ roi_depth,
                      float* __restrict__ depth_sensor) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long plane = (long long)H * W;
  if (idx < n_big) {
    const long long per = (long long)in_res * in_res;
    if (idx >= per * n) return;
    const int b = (int)(idx / per);
    const int y = (int)((idx % per) / in_res), x = (int)(idx % in_res);
    const int img = det_meta[2 * b];
    double iM[6];
    crop::invert_affine(M_in + 6 * b, iM);
    const crop::U8Tap t = crop::u8_tap(crop::src_coord(iM, x, y, false), H, W);
    const uint8_t* p00 = images + (img * plane + (long long)t.sy * W + t.sx) * C;
    const long long rowC = (long long)W * C;
    const double mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
    const long long o = (long long)b * 3 * per + (long long)y * in_res + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int cs = C == 1 ? 0 : c;   // a single-channel image is read as BGR with three equal channels
      int v = 0;
      if (t.in[0]) v += p00[cs] * t.w[0];
      if (t.in[1]) v += p00[C + cs] * t.w[1];
      if (t.in[2]) v += p00[rowC + cs] * t.w[2];
      if (t.in[3]) v += p00[rowC + C + cs] * t.w[3];
      v = crop::u8_round(v);
      roi_img[o + c * per] = __double2float_rn(__ddiv_rn(__dsub_rn((double)v, mean[c]), stdv[c]));
    }
    if (roi_depth != nullptr)
      roi_depth[(long long)b * per + (long long)y * in_res + x] = depth_nearest(depth + img * plane, H, W, iM, x, y, depth_factor[img]);
    return;
  }
  const long long j = idx - n_big;
  const long long per = (long long)out_res * out_res;
  if (j >= per * n) return;
  const int b = (int)(j / per);
  const int y = (int)((j % per) / out_res), x = (int)(j % out_res);
  double iM[6];
  crop::invert_affine(M_out + 6 * b, iM);
  const crop::F32Tap t = crop::f32_tap(crop::src_coord(iM, x, y, false), H, W);
  // the coordinate grid at the four taps, zero outside the image (the warp's constant border)
  const float gx0 = crop::grid_value(t.sx, W), gx1 = crop::grid_value(t.sx + 1, W);
  const float gy0 = crop::grid_value(t.sy, H), gy1 = crop::grid_value(t.sy + 1, H);
  const long long o = (long long)b * 2 * per + (long long)y * out_res + x;
  roi_coord_2d[o] = crop::f32_blend(t, t.in[0] ? gx0 : 0.f, t.in[1] ? gx1 : 0.f, t.in[2] ? gx0 : 0.f, t.in[3] ? gx1 : 0.f);
  roi_coord_2d[o + per] = crop::f32_blend(t, t.in[0] ? gy0 : 0.f, t.in[1] ? gy0 : 0.f, t.in[2] ? gy1 : 0.f, t.in[3] ? gy1 : 0.f);
  if (depth_sensor != nullptr) {
    // the centre 2x2 of the ROI's 4x4 cell of roi_depth, ((a + b) + (c + d)) * 0.25 in float32
    const int img = det_meta[2 * b];
    double iMi[6];
    crop::invert_affine(M_in + 6 * b, iMi);
    const uint16_t* d = depth + img * plane;
    const double f = depth_factor[img];
    const int xa = 4 * x + 1, ya = 4 * y + 1;
    const float a = depth_nearest(d, H, W, iMi, xa, ya, f), bq = depth_nearest(d, H, W, iMi, xa + 1, ya, f);
    const float c = depth_nearest(d, H, W, iMi, xa, ya + 1, f), e = depth_nearest(d, H, W, iMi, xa + 1, ya + 1, f);
    depth_sensor[(long long)b * per + (long long)y * out_res + x] = __fmul_rn(__fadd_rn(__fadd_rn(a, bq), __fadd_rn(c, e)), 0.25f);
  }
}

}  // namespace

extern "C" int gdrn_roi_setup(const int* det_meta, const float* det_xywh, int n, const float* K, const int* im_hw,
                              const float* extents, double dzi_pad_scale, int in_res, int out_res, float* roi_center,
                              float* roi_wh, float* scale, float* resize_ratio, float* roi_extent, float* roi_cam,
                              long long* roi_cls, float* im_H, float* im_W, float* bbox_xyxy, double* M_in, double* M_out,
                              void* stream) {
  GDRN_REQUIRE(n >= 0 && in_res > 0 && out_res > 0 && dzi_pad_scale > 0, "roi_setup: bad argument");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(det_meta && det_xywh && K && im_hw && extents && roi_center && roi_wh && scale && resize_ratio && roi_extent &&
                   roi_cam && roi_cls && im_H && im_W && bbox_xyxy && M_in && M_out,
               "roi_setup: null argument");
  roi_setup_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      det_meta, det_xywh, n, K, im_hw, extents, dzi_pad_scale, in_res, out_res, roi_center, roi_wh, scale, resize_ratio,
      roi_extent, roi_cam, roi_cls, im_H, im_W, bbox_xyxy, M_in, M_out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_roi_crop_multi(const uint8_t* images, int H, int W, int C, const int* det_meta, const double* M_in,
                                   const double* M_out, int n, int in_res, int out_res, const double* pixel_mean,
                                   const double* pixel_std, const uint16_t* depth, const double* depth_factor,
                                   float* roi_img, float* roi_coord_2d, float* roi_depth, float* depth_sensor, void* stream) {
  GDRN_REQUIRE(H > 0 && W > 0 && (C == 1 || C == 3) && n >= 0 && in_res > 0 && out_res > 0, "roi_crop_multi: bad shape");
  GDRN_REQUIRE(!depth_sensor || in_res == 4 * out_res, "roi_crop_multi: the sensor crop needs in_res = 4 * out_res");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(images && det_meta && M_in && M_out && pixel_mean && pixel_std && roi_img && roi_coord_2d,
               "roi_crop_multi: null argument");
  GDRN_REQUIRE(!(roi_depth || depth_sensor) || (depth && depth_factor), "roi_crop_multi: depth outputs need depth + depth_factor");
  const long long big = (long long)n * in_res * in_res, small = (long long)n * out_res * out_res;
  const long long big_blocks = (big + 255) / 256, small_blocks = (small + 255) / 256;
  roi_crop_multi_kernel<<<(unsigned)(big_blocks + small_blocks), 256, 0, (cudaStream_t)stream>>>(
      images, H, W, C, det_meta, M_in, M_out, n, in_res, out_res, big_blocks * 256, pixel_mean[0], pixel_mean[1],
      pixel_mean[2], pixel_std[0], pixel_std[1], pixel_std[2], depth, depth_factor, roi_img, roi_coord_2d, roi_depth,
      depth_sensor);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
