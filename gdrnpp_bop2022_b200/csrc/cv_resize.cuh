// cv2.resize(INTER_LINEAR) on uint8, bit-exact to OpenCV 4.x resize.cpp, shared by the YOLOX letterbox
// (yolox_letterbox.cu), the training background resize (train_aug.cu) and the YOLOX training resizes
// (yolox_train_aug.cu).  cv::resize takes one of three paths:
//   * identity (dsize == ssize): a copy;
//   * scale exactly 2 in both axes: INTER_LINEAR silently becomes the INTER_AREA fast path, (a + b + c + d + 2) >> 2;
//   * otherwise the generic fixed-point bilinear path: per output column fx = f32((dx + 0.5) * scale_x - 0.5) in float64,
//     sx = floor(fx), fx -= sx; columns left of 0 or at/after the last one are clamped with fx = 0; the weights are
//     round-half-even(f32(1 - fx) * 2048) and round-half-even(fx * 2048) (11-bit).  Rows use the same formula without
//     the clamp of fy; the two source rows are clamped to [0, H - 1] instead.  The horizontal pass sums in int, the
//     vertical one is (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2.
// scale_x / scale_y are the source-per-destination ratios cv::resize uses: 1 / (dw / W) when called with a dsize,
// 1 / fx when called with fx, fy.
#pragma once
#include "common.cuh"

namespace cvresize {

enum ResizeMode { kCopy = 0, kArea2 = 1, kLinear = 2 };

struct Tap {
  int i0, i1, w0, w1;
};

// cv::resize's coefficient table entry for output coordinate d (clamp_f: the column rule, else the row rule)
__device__ __forceinline__ Tap linear_tap(int d, double scale, int n, bool clamp_f) {
  float f = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
  int i = (int)floorf(f);
  f = __fsub_rn(f, (float)i);
  if (clamp_f) {
    if (i < 0) { f = 0.f; i = 0; }
    if (i >= n - 1) { f = 0.f; i = n - 1; }
  }
  Tap t;
  t.w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  t.w1 = __float2int_rn(__fmul_rn(f, 2048.f));
  t.i0 = min(max(i, 0), n - 1);
  t.i1 = min(max(i + 1, 0), n - 1);
  return t;
}

// The three channels of output pixel (x, y) of an H x W source (C = 1 or 3 interleaved channels, rows rowC elements
// apart; a single-channel source is read as three equal channels) under `mode`.  flip: the source is read mirrored
// left-right (source column i is img column W - 1 - i), as cv2.resize sees img[:, ::-1].
__device__ __forceinline__ void pixel_u8(const uint8_t* __restrict__ img, long long rowC, int H, int W, int C, int x, int y,
                                         int mode, double scale_x, double scale_y, int (&v)[3], bool flip = false) {
  if (mode == kCopy) {
    const uint8_t* p = img + y * rowC + (long long)(flip ? W - 1 - x : x) * C;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = p[C == 1 ? 0 : c];
  } else if (mode == kArea2) {   // the two columns swap under a flip; their sum does not change
    const uint8_t* p = img + (2LL * y) * rowC + (long long)(flip ? W - 2 - 2 * x : 2 * x) * C;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int cs = C == 1 ? 0 : c;
      v[c] = (p[cs] + p[C + cs] + p[rowC + cs] + p[rowC + C + cs] + 2) >> 2;
    }
  } else {
    const Tap tx = linear_tap(x, scale_x, W, true), ty = linear_tap(y, scale_y, H, false);
    const uint8_t* r0 = img + ty.i0 * rowC;
    const uint8_t* r1 = img + ty.i1 * rowC;
    const long long c0 = (long long)(flip ? W - 1 - tx.i0 : tx.i0) * C, c1 = (long long)(flip ? W - 1 - tx.i1 : tx.i1) * C;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int cs = C == 1 ? 0 : c;
      const int h0 = r0[c0 + cs] * tx.w0 + r0[c1 + cs] * tx.w1;
      const int h1 = r1[c0 + cs] * tx.w0 + r1[c1 + cs] * tx.w1;
      v[c] = (((ty.w0 * (h0 >> 4)) >> 16) + ((ty.w1 * (h1 >> 4)) >> 16) + 2) >> 2;
    }
  }
}

// cv::resize's path for a source of sw x sh resized to dw x dh with the given scales
__host__ __device__ __forceinline__ int resize_mode(int sh, int sw, int dh, int dw, double scale_x, double scale_y) {
  if (dh == sh && dw == sw) return kCopy;
  if (scale_x == 2.0 && scale_y == 2.0) return kArea2;
  return kLinear;
}

}  // namespace cvresize
