// Arithmetic shared by the RANSAC-voting kernels (ransac_voting.cu, ransac_layer.cu): the inlier test of
// core/csrc/ransac_voting/src/ransac_voting_kernel.cu:88-126,268-310 with the FMA contraction ptxas applies to the
// reference source spelled out (see the banner of ransac_voting.cu).
#pragma once
#include "common.cuh"

namespace {

template <bool VP>
__device__ __forceinline__ bool vote(float nx, float ny, float norm1, float cx, float cy, float hx, float hy,
                                     float hz, float thresh) {
  float dx, dy;
  if (VP) {
    dx = __fmaf_rn(-cx, hz, hx);
    dy = __fmaf_rn(-cy, hz, hy);
  } else {
    dx = __fsub_rn(hx, cx);
    dy = __fsub_rn(hy, cy);
  }
  float norm2 = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
  if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) return false;
  float den = __fmul_rn(norm1, norm2);
  if (VP) {
    float vx = __fmul_rn(nx, dx), vy = __fmul_rn(ny, dy);
    float ang = __fdiv_rn(__fadd_rn(vx, vy), den);
    if (vx < 0 || vy < 0) return false;
    return fabsf(ang) > thresh;
  } else {
    float ang = __fdiv_rn(__fmaf_rn(nx, dx, __fmul_rn(ny, dy)), den);
    return ang > thresh;
  }
}

// line-line intersection hypothesis of two pixels (ransac_voting_kernel.cu:11-49); false = degenerate pair (output stays 0)
__device__ __forceinline__ bool rv_hypothesis(float d0x, float d0y, float d1x, float d1y, float cx0, float cy0, float cx1,
                                              float cy1, float* hx, float* hy) {
  float a = __fmul_rn(d0x, d1y), b = __fmul_rn(d0y, d1x);
  float det_y = __fsub_rn(b, a);
  if ((double)fabsf(det_y) < 1e-6) return false;
  float det_x = __fsub_rn(a, b);
  if ((double)fabsf(det_x) < 1e-6) return false;
  float s1 = __fmaf_rn(d1y, cx1, -__fmul_rn(d1x, cy1));
  float s0 = __fmaf_rn(d0y, cx0, -__fmul_rn(d0x, cy0));
  float num_y = __fmaf_rn(d1y, s0, -__fmul_rn(d0y, s1));
  float num_x = __fmaf_rn(-d1x, s0, __fmul_rn(d0x, s1));
  *hx = __fdiv_rn(num_x, det_x);
  *hy = __fdiv_rn(num_y, det_y);
  return true;
}

}  // namespace
