// BOP distance images and bop19 visibility, one pixel at a time: shared by the VSD kernel (pose_error.cu) and the GT
// annotation kernel (gt_info.cu), so both restate the reference's arithmetic with the same roundings.
#pragma once
#include <cuda_runtime.h>

// misc.depth_im_to_dist_im_fast (misc.py:628-647) for one pixel: sqrt((pre_X*d)^2 + (pre_Y*d)^2 + d^2) in f64, summed
// left to right, with pre_X = (x - cx) / fx and pre_Y = (y - cy) / fy (Precomputer, misc.py:616-623).
static __device__ __forceinline__ double dist_px(double pre_x, double pre_y, float depth) {
  const double d = (double)depth;
  const double a = __dmul_rn(pre_x, d), b = __dmul_rn(pre_y, d);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(d, d)));
}

// visibility._estimate_visib_mask, bop19 mode (visibility.py:34-36): the difference is taken in f32, as the reference
// casts both distance images with astype(np.float32) and compares against delta as f32.
static __device__ __forceinline__ bool visib_bop19(double d_model, double d_test, float delta) {
  const float diff = __fsub_rn(__double2float_rn(d_model), __double2float_rn(d_test));
  return (diff <= delta || d_test == 0.0) && d_model > 0.0;
}
