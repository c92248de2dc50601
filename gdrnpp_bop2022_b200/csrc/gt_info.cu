// Ground-truth annotations of a BOP split: the per-instance math of lib/pysixd/scripts/calc_gt_info.py:110-173 and
// calc_gt_masks.py:95-113 for a batch of instances from many images, in one launch.
//
// Instance i lies in image inst_img[i]; its render on the 3x canvas (3H x 3W, principal point shifted by (W, H)) gives
// px_count_all and bbox_obj, the window [H, 2H) x [W, 2W) of that canvas gives the distance image the script compares
// with the sensor's (px_count_valid, px_count_visib, bbox_visib), and the optional image-size render gives the two
// masks of calc_gt_masks.py.  Every result is an integer: counts are summed with integer atomics and boxes are integer
// atomicMin / atomicMax over pixel coordinates, so nothing depends on the launch shape.  visib_fract is formed by the
// caller, in f64 on the host, as the script forms it.
#include <limits.h>

#include "bop_visib.cuh"
#include "common.cuh"

namespace {

constexpr int GT_THREADS = 256;
constexpr int GT_PIX_PER_THREAD = 16;
constexpr int GT_MAX_SLICES = 512;

__device__ __forceinline__ void block_reduce(unsigned (&cnt)[3], int (&box)[8], long long* counts, int* boxes) {
  __shared__ unsigned s_cnt[GT_THREADS / 32][3];
  __shared__ int s_box[GT_THREADS / 32][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 3; ++k) cnt[k] = __reduce_add_sync(0xffffffffu, cnt[k]);
#pragma unroll
  for (int k = 0; k < 8; ++k) box[k] = (k & 2) ? __reduce_max_sync(0xffffffffu, box[k]) : __reduce_min_sync(0xffffffffu, box[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) s_cnt[warp][k] = cnt[k];
#pragma unroll
    for (int k = 0; k < 8; ++k) s_box[warp][k] = box[k];
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    unsigned long long s = 0;
    for (int w = 0; w < GT_THREADS / 32; ++w) s += s_cnt[w][threadIdx.x];
    if (s) atomicAdd((unsigned long long*)counts + threadIdx.x, s);
  } else if (threadIdx.x >= 32 && threadIdx.x < 40) {
    const int k = threadIdx.x - 32;
    int v = s_box[0][k];
    for (int w = 1; w < GT_THREADS / 32; ++w) v = (k & 2) ? max(v, s_box[w][k]) : min(v, s_box[w][k]);
    if (k & 2) {
      if (v != INT_MIN) atomicMax(boxes + k, v);
    } else if (v != INT_MAX) {
      atomicMin(boxes + k, v);
    }
  }
}

// counts [n,3] = 0; boxes [n,8] = (x_min, y_min, x_max, y_max) of the canvas coverage, then of the visible mask,
// initialised empty (min = INT_MAX, max = INT_MIN)
__global__ void gt_info_init_kernel(long long* __restrict__ counts, int* __restrict__ boxes, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 8) return;
  boxes[i] = (i & 2) ? INT_MIN : INT_MAX;
  if (i < n * 3) counts[i] = 0;
}

// grid (n, slices): CTA (i, s) covers canvas pixels s*256, s*256 + slices*256, ... of instance i
__global__ void __launch_bounds__(GT_THREADS)
gt_info_kernel(const float* __restrict__ depth_large, const float* __restrict__ depth_img,
               const uint16_t* __restrict__ depth_test, const float* __restrict__ depth_scale, const double* __restrict__ Ks,
               const int* __restrict__ inst_img, int H, int W, float delta, long long* __restrict__ counts,
               int* __restrict__ boxes, uint8_t* __restrict__ mask, uint8_t* __restrict__ mask_visib) {
  const int inst = blockIdx.x, img = inst_img[inst];
  const int W3 = 3 * W;
  const long long HW = (long long)H * W, HW9 = 9 * HW;
  const float* dl = depth_large ? depth_large + (size_t)inst * HW9 : nullptr;   // null: masks only, window pixels only
  const float* di = depth_img ? depth_img + (size_t)inst * HW : nullptr;
  const uint16_t* dt = depth_test + (size_t)img * HW;
  const float scale = depth_scale[img];
  const double* K = Ks + (size_t)img * 9;
  const double fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  unsigned cnt[3] = {0u, 0u, 0u};   // px_count_all, px_count_valid, px_count_visib
  int box[8] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  const long long n_pix = dl ? HW9 : HW;
  for (long long i = (long long)blockIdx.y * GT_THREADS + threadIdx.x; i < n_pix; i += (long long)gridDim.y * GT_THREADS) {
    int y, x;
    if (dl) {
      y = (int)(i / W3);
      x = (int)(i - (long long)y * W3);
    } else {
      const int r = (int)(i / W);
      y = r + H;
      x = (int)(i - (long long)r * W) + W;
    }
    const float z = dl ? dl[i] : 0.f;
    if (z > 0.f) {   // obj_mask_gt_large = depth_gt_large > 0
      ++cnt[0];
      box[0] = min(box[0], x); box[1] = min(box[1], y); box[2] = max(box[2], x); box[3] = max(box[3], y);
    }
    const int wy = y - H, wx = x - W;
    if (wy < 0 || wy >= H || wx < 0 || wx >= W) continue;
    const size_t p = (size_t)wy * W + wx;
    const float zi = di ? di[p] : 0.f;
    if (z == 0.f && zi == 0.f) {   // dist 0: in no mask and not valid
      if (di) { mask[(size_t)inst * HW + p] = 0; mask_visib[(size_t)inst * HW + p] = 0; }
      continue;
    }
    const double pre_x = __ddiv_rn(__dsub_rn((double)wx, cx), fx);
    const double pre_y = __ddiv_rn(__dsub_rn((double)wy, cy), fy);
    const double dist_im = dist_px(pre_x, pre_y, __fmul_rn((float)dt[p], scale));   // depth *= depth_scale, in f32
    if (z != 0.f) {
      const double dist_gt = dist_px(pre_x, pre_y, z);
      cnt[1] += (dist_gt > 0.0 && dist_im > 0.0);
      if (visib_bop19(dist_gt, dist_im, delta)) {
        ++cnt[2];
        box[4] = min(box[4], wx); box[5] = min(box[5], wy); box[6] = max(box[6], wx); box[7] = max(box[7], wy);
      }
    }
    if (di) {   // calc_gt_masks.py: mask = dist_gt > 0, mask_visib = bop19 visibility, both as 0 / 255
      const double dist_g2 = dist_px(pre_x, pre_y, zi);
      mask[(size_t)inst * HW + p] = dist_g2 > 0.0 ? 255 : 0;
      mask_visib[(size_t)inst * HW + p] = visib_bop19(dist_g2, dist_im, delta) ? 255 : 0;
    }
  }
  block_reduce(cnt, box, counts + (size_t)inst * 3, boxes + (size_t)inst * 8);
}

// calc_2d_bbox (x, y, x_max - x_min, y_max - y_min), the canvas box shifted back by (W, H); both boxes are
// [-1, -1, -1, -1] unless px_count_visib > 0 (calc_gt_info.py:141-154)
__global__ void gt_info_finalize_kernel(const long long* __restrict__ counts, int* __restrict__ boxes, int n, int H, int W) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int* b = boxes + (size_t)i * 8;
  if (counts[(size_t)i * 3 + 2] == 0) {
    for (int k = 0; k < 8; ++k) b[k] = -1;
    return;
  }
  const int ox0 = b[0], oy0 = b[1], ox1 = b[2], oy1 = b[3], vx0 = b[4], vy0 = b[5], vx1 = b[6], vy1 = b[7];
  b[0] = ox0 - W; b[1] = oy0 - H; b[2] = ox1 - ox0; b[3] = oy1 - oy0;
  b[4] = vx0; b[5] = vy0; b[6] = vx1 - vx0; b[7] = vy1 - vy0;
}

}  // namespace

extern "C" int gdrn_gt_info(const float* depth_large, const float* depth_img, const uint16_t* depth_test,
                            const float* depth_scale, const double* Ks, const int* inst_img, int n, int H, int W,
                            float delta, long long* counts, int* boxes, uint8_t* mask, uint8_t* mask_visib, void* stream) {
  GDRN_REQUIRE(depth_test && depth_scale && Ks && inst_img && counts && boxes, "gt_info: null argument");
  GDRN_REQUIRE(depth_large || depth_img, "gt_info: need depth_large, depth_img or both");
  GDRN_REQUIRE(!depth_img || (mask && mask_visib), "gt_info: depth_img needs both mask outputs");
  GDRN_REQUIRE(n > 0 && H > 0 && W > 0, "gt_info: need n, H, W > 0");
  GDRN_REQUIRE((long long)H * 3 <= INT_MAX / 3 / W, "gt_info: canvas too large");
  cudaStream_t st = (cudaStream_t)stream;
  gt_info_init_kernel<<<(n * 8 + 255) / 256, 256, 0, st>>>(counts, boxes, n);
  const long long HW9 = (depth_large ? 9LL : 1LL) * H * W;
  const int slices = (int)min((HW9 + GT_THREADS * GT_PIX_PER_THREAD - 1) / (GT_THREADS * GT_PIX_PER_THREAD),
                              (long long)GT_MAX_SLICES);
  gt_info_kernel<<<dim3(n, slices), GT_THREADS, 0, st>>>(depth_large, depth_img, depth_test, depth_scale, Ks, inst_img, H,
                                                         W, delta, counts, boxes, depth_img ? mask : nullptr,
                                                         depth_img ? mask_visib : nullptr);
  gt_info_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(counts, boxes, n, H, W);
  gdrn_count_launch(3);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gdrn_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
    return GDRN_ERR_CUDA;
  }
  return 0;
}
