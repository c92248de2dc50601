// ROI crop + resize on the GPU (SURVEY.md 8f rank 1): the reference crops every ROI with
// crop_resize_by_warp_affine = cv2.warpAffine (core/utils/data_utils.py:115-133), one ROI at a time on the host
// (demo/predictor_gdrn.py:417-438; datasets/data_loader.py:758-797), for the image (uint8, bilinear, then
// normalize_image), the 2-D coordinate grid (float, bilinear, 64x64) and the depth crop (float, nearest).
// These kernels reproduce OpenCV's warpAffine arithmetic exactly (the CPU restatement used by the tests is
// pinned against cv2 itself): double-precision inverse of the forward matrix, 10-bit fixed-point source coordinates
// built from cvRound()ed per-column / per-row terms, 5 fractional bits, 15-bit integer bilinear weights with the
// (32767, 0, 0, 1) quirk at integer positions, (sum + 2^14) >> 15, zero border.  One thread per output pixel; the
// uint8 path writes the normalised NCHW fp32 crop the stem kernel consumes.  Memory-bound: 12 B written per pixel.
#include "crop_common.cuh"

namespace {

using crop::SrcCoord;

__global__ void __launch_bounds__(256)
crop_resize_u8_kernel(const uint8_t* __restrict__ img, int H, int W, int C, const double* __restrict__ Ms, int n, int oh,
                      int ow, double m0, double m1, double m2, double s0, double s1, double s2, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = (long long)oh * ow;
  if (idx >= per * n) return;
  const int b = (int)(idx / per);
  const int y = (int)((idx % per) / ow), x = (int)(idx % ow);
  double iM[6];
  crop::invert_affine(Ms + 6 * b, iM);
  const crop::U8Tap t = crop::u8_tap(crop::src_coord(iM, x, y, false), H, W);
  const uint8_t* p00 = img + ((long long)t.sy * W + t.sx) * C;
  const double mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
  for (int c = 0; c < C; ++c) {
    int v = 0;
    if (t.in[0]) v += p00[c] * t.w[0];
    if (t.in[1]) v += p00[C + c] * t.w[1];
    if (t.in[2]) v += p00[(long long)W * C + c] * t.w[2];
    if (t.in[3]) v += p00[(long long)W * C + C + c] * t.w[3];
    v = crop::u8_round(v);
    // normalize_image: (uint8 - mean) / std in float64, then astype(float32) (predictor_gdrn.py normalize_image)
    const int cc = c < 3 ? c : 2;
    out[((long long)b * C + c) * per + (long long)y * ow + x] = __double2float_rn(__ddiv_rn(__dsub_rn((double)v, mean[cc]), stdv[cc]));
  }
}

__global__ void __launch_bounds__(256)
crop_resize_f32_kernel(const float* __restrict__ src, int H, int W, int C, const double* __restrict__ Ms, int n, int oh,
                       int ow, int nearest, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = (long long)oh * ow;
  if (idx >= per * n) return;
  const int b = (int)(idx / per);
  const int y = (int)((idx % per) / ow), x = (int)(idx % ow);
  double iM[6];
  crop::invert_affine(Ms + 6 * b, iM);
  const SrcCoord sc = crop::src_coord(iM, x, y, nearest != 0);
  float* o = out + (long long)b * C * per + (long long)y * ow + x;
  if (nearest) {
    const bool in = sc.X >= 0 && sc.X < W && sc.Y >= 0 && sc.Y < H;
    for (int c = 0; c < C; ++c) o[c * per] = in ? src[((long long)sc.Y * W + sc.X) * C + c] : 0.f;
    return;
  }
  const crop::F32Tap t = crop::f32_tap(sc, H, W);
  const float* p00 = src + ((long long)t.sy * W + t.sx) * C;
  for (int c = 0; c < C; ++c) {
    const float a = t.in[0] ? p00[c] : 0.f, bq = t.in[1] ? p00[C + c] : 0.f;
    const float cq = t.in[2] ? p00[(long long)W * C + c] : 0.f, d = t.in[3] ? p00[(long long)W * C + C + c] : 0.f;
    o[c * per] = crop::f32_blend(t, a, bq, cq, d);
  }
}

}  // namespace

extern "C" int gdrn_crop_resize_u8(const uint8_t* image, int H, int W, int C, const double* M, int n, int out_h, int out_w,
                                   const double* pixel_mean, const double* pixel_std, float* out, void* stream) {
  GDRN_REQUIRE(H > 0 && W > 0 && C >= 1 && C <= 4 && n >= 0 && out_h > 0 && out_w > 0, "crop_resize_u8: bad shape");
  if (n == 0) return GDRN_OK;   // empty detection list: nothing to do (the reference loop simply does not iterate)
  GDRN_REQUIRE(image && M && out && pixel_mean && pixel_std, "crop_resize_u8: null argument");
  const long long total = (long long)n * out_h * out_w;
  const double* mu = pixel_mean;
  const double* sd = pixel_std;
  crop_resize_u8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      image, H, W, C, M, n, out_h, out_w, mu[0], mu[C > 1 ? 1 : 0], mu[C > 2 ? 2 : 0], sd[0], sd[C > 1 ? 1 : 0],
      sd[C > 2 ? 2 : 0], out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_crop_resize_f32(const float* src, int H, int W, int C, const double* M, int n, int out_h, int out_w,
                                    int nearest, float* out, void* stream) {
  GDRN_REQUIRE(H > 0 && W > 0 && C >= 1 && n >= 0 && out_h > 0 && out_w > 0, "crop_resize_f32: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(src && M && out, "crop_resize_f32: null argument");
  const long long total = (long long)n * out_h * out_w;
  crop_resize_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(src, H, W, C, M, n, out_h, out_w,
                                                                                       nearest, out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
