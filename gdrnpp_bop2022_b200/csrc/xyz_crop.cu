// The xyz_crop training targets of a BOP split (the reference's *_1_gen_xyz.py scripts, e.g.
// core/gdrn_modeling/tools/tless/tless_pbr_1_gen_xyz.py) for many instances in two launches.
//
// Each instance is rendered alone (float z, 0 = background).  gdrn_xyz_crop_boxes finds the inclusive pixel box of its
// coverage (depth != 0); the host reads the boxes back, sizes one packed buffer from them and gdrn_xyz_crop_pack
// back-projects the pixels inside each box as misc.calc_xyz_bp_torch does, in fp32:
//   xc = ((u - cx) * z) / fx,  yc = ((v - cy) * z) / fy,  zc = z,  xyz = R^T ((xc, yc, zc) - t),  0 where z == 0,
// and stores the crop as fp16 (round to nearest even) [h,w,3] row-major at the instance's offset.  The camera-space step
// rounds the product before the division, as torch does (no fma); the rotation is a dot product whose order the
// reference leaves to cuBLAS.  Boxes are integer min / max reductions, so nothing depends on the launch shape.
#include <cuda_fp16.h>
#include <limits.h>

#include "common.cuh"

namespace {

constexpr int XYZ_THREADS = 256;
constexpr int XYZ_PIX_PER_THREAD = 16;
constexpr int XYZ_MAX_SLICES = 512;
constexpr int XYZ_PACK_SLICES = 32;

__global__ void xyz_boxes_init_kernel(int* __restrict__ boxes, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n * 4) boxes[i] = (i & 2) ? INT_MIN : INT_MAX;
}

// grid (n, slices): CTA (i, s) covers pixels s*256, s*256 + slices*256, ... of render i; one atomic per box field per CTA
__global__ void __launch_bounds__(XYZ_THREADS)
xyz_boxes_kernel(const float* __restrict__ depth, int H, int W, int* __restrict__ boxes) {
  __shared__ int s_box[XYZ_THREADS / 32][4];
  const int inst = blockIdx.x;
  const long long HW = (long long)H * W;
  const float* d = depth + (size_t)inst * HW;
  int box[4] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  for (long long i = (long long)blockIdx.y * XYZ_THREADS + threadIdx.x; i < HW; i += (long long)gridDim.y * XYZ_THREADS) {
    if (d[i] != 0.f) {
      const int y = (int)(i / W), x = (int)(i - (long long)y * W);
      box[0] = min(box[0], x); box[1] = min(box[1], y); box[2] = max(box[2], x); box[3] = max(box[3], y);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 4; ++k) box[k] = (k & 2) ? __reduce_max_sync(0xffffffffu, box[k]) : __reduce_min_sync(0xffffffffu, box[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) s_box[warp][k] = box[k];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    const int k = threadIdx.x;
    int v = s_box[0][k];
    for (int w = 1; w < XYZ_THREADS / 32; ++w) v = (k & 2) ? max(v, s_box[w][k]) : min(v, s_box[w][k]);
    if (k & 2) {
      if (v != INT_MIN) atomicMax(boxes + (size_t)inst * 4 + k, v);
    } else if (v != INT_MAX) {
      atomicMin(boxes + (size_t)inst * 4 + k, v);
    }
  }
}

// grid (n, XYZ_PACK_SLICES): CTA (i, s) strides over the pixels of instance i's box (the whole frame, as zeros, when the
// render is empty) and writes their three fp16 components
__global__ void __launch_bounds__(XYZ_THREADS)
xyz_pack_kernel(const float* __restrict__ depth, const float* __restrict__ R, const float* __restrict__ t,
                const float* __restrict__ K, const int* __restrict__ boxes, const long long* __restrict__ offsets, int H,
                int W, __half* __restrict__ out) {
  const int inst = blockIdx.x;
  const int* b = boxes + (size_t)inst * 4;
  const bool empty = b[0] > b[2];
  const int x1 = empty ? 0 : b[0], y1 = empty ? 0 : b[1];
  const int bw = empty ? W : b[2] - b[0] + 1, bh = empty ? H : b[3] - b[1] + 1;
  const long long npx = (long long)bw * bh;
  __half* o = out + offsets[inst];
  const __half zero = __float2half_rn(0.f);
  if (empty) {
    for (long long i = (long long)blockIdx.y * XYZ_THREADS + threadIdx.x; i < npx * 3; i += (long long)gridDim.y * XYZ_THREADS)
      o[i] = zero;
    return;
  }
  const float* d = depth + (size_t)inst * H * W;
  const float* Ri = R + (size_t)inst * 9;
  const float* ti = t + (size_t)inst * 3;
  const float* Ki = K + (size_t)inst * 9;
  const float fx = Ki[0], cx = Ki[2], fy = Ki[4], cy = Ki[5];
  const float r00 = Ri[0], r01 = Ri[1], r02 = Ri[2], r10 = Ri[3], r11 = Ri[4], r12 = Ri[5], r20 = Ri[6], r21 = Ri[7],
              r22 = Ri[8];
  const float tx = ti[0], ty = ti[1], tz = ti[2];
  for (long long i = (long long)blockIdx.y * XYZ_THREADS + threadIdx.x; i < npx; i += (long long)gridDim.y * XYZ_THREADS) {
    const int yy = (int)(i / bw), xx = (int)(i - (long long)yy * bw);
    const int u = x1 + xx, v = y1 + yy;
    const float z = d[(size_t)v * W + u];
    __half hx = zero, hy = zero, hz = zero;
    if (z != 0.f) {
      const float xc = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, cx), z), fx);
      const float yc = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, cy), z), fy);
      const float dx = __fsub_rn(xc, tx), dy = __fsub_rn(yc, ty), dz = __fsub_rn(z, tz);
      hx = __float2half_rn(fmaf(r20, dz, fmaf(r10, dy, __fmul_rn(r00, dx))));
      hy = __float2half_rn(fmaf(r21, dz, fmaf(r11, dy, __fmul_rn(r01, dx))));
      hz = __float2half_rn(fmaf(r22, dz, fmaf(r12, dy, __fmul_rn(r02, dx))));
    }
    o[i * 3] = hx; o[i * 3 + 1] = hy; o[i * 3 + 2] = hz;
  }
}

}  // namespace

extern "C" int gdrn_xyz_crop_boxes(const float* depth, int n, int H, int W, int* boxes, void* stream) {
  GDRN_REQUIRE(depth && boxes, "xyz_crop_boxes: null argument");
  GDRN_REQUIRE(n > 0 && H > 0 && W > 0, "xyz_crop_boxes: need n, H, W > 0");
  GDRN_REQUIRE((long long)H * W <= INT_MAX, "xyz_crop_boxes: image too large");
  cudaStream_t st = (cudaStream_t)stream;
  xyz_boxes_init_kernel<<<(n * 4 + 255) / 256, 256, 0, st>>>(boxes, n);
  const long long HW = (long long)H * W;
  const int slices = (int)min((HW + XYZ_THREADS * XYZ_PIX_PER_THREAD - 1) / (XYZ_THREADS * XYZ_PIX_PER_THREAD),
                              (long long)XYZ_MAX_SLICES);
  xyz_boxes_kernel<<<dim3(n, slices), XYZ_THREADS, 0, st>>>(depth, H, W, boxes);
  gdrn_count_launch(2);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gdrn_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
    return GDRN_ERR_CUDA;
  }
  return 0;
}

extern "C" int gdrn_xyz_crop_pack(const float* depth, const float* R, const float* t, const float* K, const int* boxes,
                                  const long long* offsets, int n, int H, int W, uint16_t* out, void* stream) {
  GDRN_REQUIRE(depth && R && t && K && boxes && offsets && out, "xyz_crop_pack: null argument");
  GDRN_REQUIRE(n > 0 && H > 0 && W > 0, "xyz_crop_pack: need n, H, W > 0");
  GDRN_REQUIRE((long long)H * W <= INT_MAX / 3, "xyz_crop_pack: image too large");
  xyz_pack_kernel<<<dim3(n, XYZ_PACK_SLICES), XYZ_THREADS, 0, (cudaStream_t)stream>>>(depth, R, t, K, boxes, offsets, H, W,
                                                                                      reinterpret_cast<__half*>(out));
  gdrn_count_launch(1);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gdrn_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
    return GDRN_ERR_CUDA;
  }
  return 0;
}
