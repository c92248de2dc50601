// OpenCV warpAffine arithmetic shared by the single-image crops (crop_resize.cu) and the batched ROI inputs
// (roi_batch.cu): double-precision inverse of the forward matrix, 10-bit fixed-point source coordinates built from
// cvRound()ed per-column / per-row terms, 5 fractional bits, and the two bilinear weight sets (15-bit integer for
// uint8, float for float sources).  Every double / float operation carries explicit rounding: nvcc must not contract
// a*b+c into an FMA (OpenCV's host code does not).
#pragma once
#include "common.cuh"

namespace crop {

struct SrcCoord { int X, Y; };

__device__ __forceinline__ void invert_affine(const double* __restrict__ M, double (&iM)[6]) {
  double D = __dsub_rn(__dmul_rn(M[0], M[4]), __dmul_rn(M[1], M[3]));
  D = D != 0 ? __ddiv_rn(1.0, D) : 0.0;
  const double A11 = __dmul_rn(M[4], D), A22 = __dmul_rn(M[0], D);
  iM[0] = A11; iM[1] = __dmul_rn(M[1], -D); iM[3] = __dmul_rn(M[3], -D); iM[4] = A22;
  iM[2] = __dsub_rn(__dmul_rn(-iM[0], M[2]), __dmul_rn(iM[1], M[5]));
  iM[5] = __dsub_rn(__dmul_rn(-iM[3], M[2]), __dmul_rn(iM[4], M[5]));
}

// nearest: the integer source pixel; bilinear: source position in 1/32 pixel
__device__ __forceinline__ SrcCoord src_coord(const double (&iM)[6], int x, int y, bool nearest) {
  constexpr int AB_BITS = 10, AB_SCALE = 1 << 10, INTER_BITS = 5;
  const int round_delta = nearest ? AB_SCALE / 2 : AB_SCALE / 32 / 2;
  const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(iM[0], (double)x), (double)AB_SCALE));
  const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(iM[3], (double)x), (double)AB_SCALE));
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(iM[1], (double)y), iM[2]), (double)AB_SCALE)) + round_delta;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(iM[4], (double)y), iM[5]), (double)AB_SCALE)) + round_delta;
  SrcCoord c;
  const int sh = nearest ? AB_BITS : AB_BITS - INTER_BITS;
  c.X = (X0 + adelta) >> sh;
  c.Y = (Y0 + bdelta) >> sh;
  return c;
}

__device__ __forceinline__ int sat_short(int v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }

// uint8 bilinear tap: top-left source pixel (saturated like OpenCV's short map), 15-bit weights (exact products of the
// 1/32 fractions; saturate_cast<short>(32768) = 32767, deficit to weight 3) and which of the four taps lie inside
struct U8Tap { int sx, sy; int w[4]; bool in[4]; };

__device__ __forceinline__ U8Tap u8_tap(SrcCoord sc, int H, int W) {
  U8Tap t;
  t.sx = sat_short(sc.X >> 5); t.sy = sat_short(sc.Y >> 5);
  const int fx = sc.X & 31, fy = sc.Y & 31;
  t.w[0] = (32 - fy) * (32 - fx) * 32; t.w[1] = (32 - fy) * fx * 32; t.w[2] = fy * (32 - fx) * 32; t.w[3] = fy * fx * 32;
  if (t.w[0] > 32767) { t.w[0] = 32767; t.w[3] += 1; }
  const bool x0 = t.sx >= 0 && t.sx < W, x1 = t.sx + 1 >= 0 && t.sx + 1 < W;
  const bool y0 = t.sy >= 0 && t.sy < H, y1 = t.sy + 1 >= 0 && t.sy + 1 < H;
  t.in[0] = x0 && y0; t.in[1] = x1 && y0; t.in[2] = x0 && y1; t.in[3] = x1 && y1;
  return t;
}

// (sum + 2^14) >> 15, clamped to [0, 255]
__device__ __forceinline__ int u8_round(int v) {
  v = (v + (1 << 14)) >> 15;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// float bilinear tap (no saturation of the source position, as OpenCV's float remap)
struct F32Tap { int sx, sy; float w[4]; bool in[4]; };

__device__ __forceinline__ F32Tap f32_tap(SrcCoord sc, int H, int W) {
  F32Tap t;
  t.sx = sc.X >> 5; t.sy = sc.Y >> 5;
  const float ax = (float)(sc.X & 31) * (1.f / 32), ay = (float)(sc.Y & 31) * (1.f / 32);
  t.w[0] = __fmul_rn(1.f - ay, 1.f - ax); t.w[1] = __fmul_rn(1.f - ay, ax); t.w[2] = __fmul_rn(ay, 1.f - ax); t.w[3] = __fmul_rn(ay, ax);
  const bool x0 = t.sx >= 0 && t.sx < W, x1 = t.sx + 1 >= 0 && t.sx + 1 < W;
  const bool y0 = t.sy >= 0 && t.sy < H, y1 = t.sy + 1 >= 0 && t.sy + 1 < H;
  t.in[0] = x0 && y0; t.in[1] = x1 && y0; t.in[2] = x0 && y1; t.in[3] = x1 && y1;
  return t;
}

// same association as OpenCV's scalar remapBilinear: ((a*w0 + b*w1) + c*w2) + d*w3, no FMA
__device__ __forceinline__ float f32_blend(const F32Tap& t, float a, float b, float c, float d) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, t.w[0]), __fmul_rn(b, t.w[1])), __fmul_rn(c, t.w[2])), __fmul_rn(d, t.w[3]));
}

}  // namespace crop
