// Pose visualisation composite: the pixel arithmetic of visualization.vis_object_poses
// (lib/pysixd/visualization.py:155-258) for a batch of images, each with its instance renders, in one pass set.
//
// Image j owns instances [inst_off[j], inst_off[j+1]) in drawing order.  Per pixel, in that order:
//   resolve:      m_mask = m_depth != 0 && (ren_depth == 0 || m_depth < ren_depth); ren_rgb/ren_depth take the
//                 instance where m_mask holds (nearest wins, the first one on equal depth)
//   non-resolve:  ren_rgb = min(255, ren_rgb + m_rgb)   (the saturating u8 sum)
//   blend = floor(0.5 * rgb + 0.5 * ren_rgb), which is (rgb + ren_rgb) >> 1.  The reference adds the integer info
//   layer to 0.5*rgb + 0.5*ren_rgb in f32 and truncates; that equals this blend plus the layer, clipped at 255.
//   boxes [n,4] = x_min, y_min, x_max, y_max of each instance's own m_rgb > 0 (INT_MAX / INT_MIN when empty), from
//   warp reductions, shared-memory atomics per CTA and one global atomic set per CTA and instance: integers, so they
//   do not depend on the launch shape.
// Depth difference (f32 as the reference): valid = depth > 0 && ren_depth > 0, diff = valid ? ren_depth - depth : 0,
//   R = 255 * (valid && diff < 15); x = diff - min(diff over ALL pixels); over mask = x > 0, in f64:
//   G = B = trunc(255 * ((x - min_mask) / ((max_mask - min_mask) / 0.8) + 0.2)) (depth_for_vis), 0 where !valid.
//   An empty mask gives G = B = 0; max_mask == min_mask gives 0/0, taken as 0 (51).
//   stats per image: min, max of diff[valid] (f32), their f64 sum (summed in a fixed order) and count.
#include <limits.h>

#include "common.cuh"

namespace {

constexpr int VP_THREADS = 256;
constexpr int VP_PIX_PER_THREAD = 8;
constexpr int VP_MAX_SLICES = 256;
constexpr int VP_MAX_INST = 3000;   // instances of one image: their boxes (16 B each) fit the default 48 KB of shared memory
constexpr int VP_RGB = 1, VP_RESOLVE = 2, VP_DEPTH_DIFF = 4;

// monotone map of an f32 to a signed int (and back: the map is its own inverse), so that integer atomicMin/Max order
// floats of either sign
__device__ __forceinline__ int f2ord(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

struct VisStats {        // per image
  int gmin;              // f2ord(min of diff over all pixels)
  int vmin, vmax;        // f2ord(min / max of diff[valid])
  int mmin, mmax;        // f2ord(min / max of x over x > 0)
  unsigned long long count;
};

__global__ void vis_init_kernel(VisStats* __restrict__ st, int N, int* __restrict__ boxes, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) st[i] = VisStats{INT_MAX, INT_MAX, INT_MIN, INT_MAX, INT_MIN, 0ull};
  if (boxes && i < n * 4) boxes[i] = (i & 2) ? INT_MIN : INT_MAX;
}

template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = sh[0];
  for (int w = 1; w < VP_THREADS / 32; ++w) v = op(v, sh[w]);
  return v;
}

struct MinI { __device__ int operator()(int a, int b) const { return min(a, b); } };
struct MaxI { __device__ int operator()(int a, int b) const { return max(a, b); } };
struct AddD { __device__ double operator()(double a, double b) const { return a + b; } };
struct AddU { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; } };

// grid (slices, N): CTA (s, j) covers pixels s*256 + k*slices*256 of image j (a uniform trip count per warp)
__global__ void __launch_bounds__(VP_THREADS)
vis_composite_kernel(const uint8_t* __restrict__ m_rgb, const float* __restrict__ m_depth, const int* __restrict__ inst_off,
                     const uint8_t* __restrict__ rgb, const float* __restrict__ depth, int H, int W, int flags,
                     uint8_t* __restrict__ ren_rgb, float* __restrict__ ren_depth, uint8_t* __restrict__ blend,
                     int* __restrict__ boxes, float* __restrict__ diff, VisStats* __restrict__ st,
                     double* __restrict__ sum_part) {
  const int j = blockIdx.y, k0 = inst_off[j], k1 = inst_off[j + 1];
  const long long HW = (long long)H * W;
  const bool do_rgb = flags & VP_RGB, resolve = flags & VP_RESOLVE, do_diff = flags & VP_DEPTH_DIFF;
  const bool need_depth = do_diff || (do_rgb && resolve);
  const int lane = threadIdx.x & 31;
  extern __shared__ int s_box[];   // [k1 - k0][4]: this CTA's boxes, flushed to boxes with one atomic set per instance
  if (do_rgb)
    for (int i = threadIdx.x; i < (k1 - k0) * 4; i += VP_THREADS) s_box[i] = (i & 2) ? INT_MIN : INT_MAX;
  __syncthreads();
  int gmin = INT_MAX, vmin = INT_MAX, vmax = INT_MIN;
  unsigned long long cnt = 0;
  double sum = 0.0;
  const long long stride = (long long)gridDim.x * VP_THREADS;
  for (long long base = (long long)blockIdx.x * VP_THREADS; base < HW; base += stride) {
    const long long p = base + threadIdx.x;
    const bool inb = p < HW;
    const int y = inb ? (int)(p / W) : 0, x = inb ? (int)(p - (long long)y * W) : 0;
    float rd = 0.f;
    int rr = 0, rg = 0, rb = 0;
    for (int k = k0; k < k1; ++k) {
      const size_t q = (size_t)k * HW + p;
      const float md = (inb && need_depth) ? m_depth[q] : 0.f;
      const bool vis = md != 0.f && (rd == 0.f || md < rd);
      if (vis) rd = md;
      if (!do_rgb) continue;
      int mr = 0, mg = 0, mb = 0;
      if (inb) { mr = m_rgb[q * 3]; mg = m_rgb[q * 3 + 1]; mb = m_rgb[q * 3 + 2]; }
      if (resolve) {
        if (vis) { rr = mr; rg = mg; rb = mb; }
      } else {
        rr = min(255, rr + mr); rg = min(255, rg + mg); rb = min(255, rb + mb);
      }
      const bool on = (mr | mg | mb) != 0;
      if (__ballot_sync(0xffffffffu, on)) {
        const int bx0 = __reduce_min_sync(0xffffffffu, on ? x : INT_MAX), by0 = __reduce_min_sync(0xffffffffu, on ? y : INT_MAX);
        const int bx1 = __reduce_max_sync(0xffffffffu, on ? x : INT_MIN), by1 = __reduce_max_sync(0xffffffffu, on ? y : INT_MIN);
        if (lane == 0) {
          int* b = s_box + (k - k0) * 4;
          atomicMin(b, bx0); atomicMin(b + 1, by0); atomicMax(b + 2, bx1); atomicMax(b + 3, by1);
        }
      }
    }
    if (!inb) continue;
    const size_t o = (size_t)j * HW + p;
    if (need_depth) ren_depth[o] = rd;
    if (do_rgb) {
      ren_rgb[o * 3] = (uint8_t)rr; ren_rgb[o * 3 + 1] = (uint8_t)rg; ren_rgb[o * 3 + 2] = (uint8_t)rb;
      blend[o * 3] = (uint8_t)((rgb[o * 3] + rr) >> 1);
      blend[o * 3 + 1] = (uint8_t)((rgb[o * 3 + 1] + rg) >> 1);
      blend[o * 3 + 2] = (uint8_t)((rgb[o * 3 + 2] + rb) >> 1);
    }
    if (do_diff) {
      const float d = depth[o];
      const bool valid = d > 0.f && rd > 0.f;
      const float df = valid ? __fsub_rn(rd, d) : 0.f;
      diff[o] = df;
      gmin = min(gmin, f2ord(df));
      if (valid) {
        vmin = min(vmin, f2ord(df)); vmax = max(vmax, f2ord(df));
        ++cnt;
        sum += (double)df;
      }
    }
  }
  if (do_rgb) {
    __syncthreads();
    for (int i = threadIdx.x; i < (k1 - k0) * 4; i += VP_THREADS) {
      const int v = s_box[i];
      if (i & 2) {
        if (v != INT_MIN) atomicMax(boxes + k0 * 4 + i, v);
      } else if (v != INT_MAX) {
        atomicMin(boxes + k0 * 4 + i, v);
      }
    }
  }
  if (!do_diff) return;
  __shared__ int sh_i[VP_THREADS / 32];
  __shared__ double sh_d[VP_THREADS / 32];
  __shared__ unsigned long long sh_u[VP_THREADS / 32];
  gmin = block_reduce(gmin, MinI(), sh_i);
  vmin = block_reduce(vmin, MinI(), sh_i);
  vmax = block_reduce(vmax, MaxI(), sh_i);
  cnt = block_reduce(cnt, AddU(), sh_u);
  sum = block_reduce(sum, AddD(), sh_d);
  if (threadIdx.x == 0) {
    VisStats* s = st + j;
    atomicMin(&s->gmin, gmin);
    if (cnt) { atomicMin(&s->vmin, vmin); atomicMax(&s->vmax, vmax); atomicAdd(&s->count, cnt); }
    sum_part[(size_t)j * gridDim.x + blockIdx.x] = sum;
  }
}

// masked min / max of x = diff - gmin over x > 0 (depth_for_vis' mask); CTA (0, j) also sums image j's partial sums
// in slice order, so the f64 sum does not depend on which CTA finished first
__global__ void __launch_bounds__(VP_THREADS)
vis_diff_range_kernel(const float* __restrict__ diff, int H, int W, VisStats* __restrict__ st,
                      const double* __restrict__ sum_part, float* __restrict__ minmax, double* __restrict__ sums,
                      long long* __restrict__ counts) {
  const int j = blockIdx.y;
  const long long HW = (long long)H * W;
  const float gmin = ord2f(st[j].gmin);
  int mn = INT_MAX, mx = INT_MIN;
  for (long long p = (long long)blockIdx.x * VP_THREADS + threadIdx.x; p < HW; p += (long long)gridDim.x * VP_THREADS) {
    const float x = __fsub_rn(diff[(size_t)j * HW + p], gmin);
    if (x > 0.f) { mn = min(mn, __float_as_int(x)); mx = max(mx, __float_as_int(x)); }   // positive: bits are ordered
  }
  __shared__ int sh_i[VP_THREADS / 32];
  mn = block_reduce(mn, MinI(), sh_i);
  mx = block_reduce(mx, MaxI(), sh_i);
  if (threadIdx.x == 0) {
    if (mx != INT_MIN) { atomicMin(&st[j].mmin, f2ord(__int_as_float(mn))); atomicMax(&st[j].mmax, f2ord(__int_as_float(mx))); }
    if (blockIdx.x == 0) {   // diff[valid] statistics, read by the host for the text lines
      double s = 0.0;
      for (int k = 0; k < (int)gridDim.x; ++k) s += sum_part[(size_t)j * gridDim.x + k];
      sums[j] = s;
      counts[j] = (long long)st[j].count;
      minmax[j * 2] = ord2f(st[j].vmin);
      minmax[j * 2 + 1] = ord2f(st[j].vmax);
    }
  }
}

__global__ void __launch_bounds__(VP_THREADS)
vis_diff_image_kernel(const float* __restrict__ diff, const float* __restrict__ ren_depth, const float* __restrict__ depth,
                      int H, int W, const VisStats* __restrict__ st, uint8_t* __restrict__ diff_vis) {
  const int j = blockIdx.y;
  const long long HW = (long long)H * W;
  const VisStats s = st[j];
  const float gmin = ord2f(s.gmin);
  const bool any = s.mmax != INT_MIN;
  const double mn = any ? (double)ord2f(s.mmin) : 0.0;
  const double range = any ? __dsub_rn((double)ord2f(s.mmax), mn) : 0.0;
  const double div = __ddiv_rn(range, 1.0 - 0.2);
  for (long long p = (long long)blockIdx.x * VP_THREADS + threadIdx.x; p < HW; p += (long long)gridDim.x * VP_THREADS) {
    const size_t o = (size_t)j * HW + p;
    const float df = diff[o];
    uint8_t r = 0, g = 0;
    if (depth[o] > 0.f && ren_depth[o] > 0.f) {
      r = df < 15.f ? 255 : 0;
      const float x = __fsub_rn(df, gmin);
      if (x > 0.f) {
        const double a = __dsub_rn((double)x, mn);
        const double q = range == 0.0 ? 0.0 : __ddiv_rn(a, div);
        g = (uint8_t)__dmul_rn(255.0, __dadd_rn(q, 0.2));
      }
    }
    diff_vis[o * 3] = r; diff_vis[o * 3 + 1] = g; diff_vis[o * 3 + 2] = g;
  }
}

}  // namespace

// workspace: per-image stats (256-byte aligned head), per-(image, slice) partial sums, the diff image
static size_t vis_stats_bytes(int N) { return ((size_t)N * sizeof(VisStats) + 255) / 256 * 256; }

extern "C" size_t gdrn_vis_poses_workspace_bytes(int N, int H, int W) {
  return vis_stats_bytes(N) + (size_t)N * VP_MAX_SLICES * 8 + (size_t)N * H * W * 4;
}

extern "C" int gdrn_vis_poses(const uint8_t* m_rgb, const float* m_depth, const int* inst_off, int max_inst, int N, int n,
                              const uint8_t* rgb, const float* depth, int H, int W, int flags, uint8_t* ren_rgb,
                              float* ren_depth, uint8_t* blend, int* boxes, uint8_t* diff_vis, float* diff_minmax,
                              double* diff_sum, long long* diff_count, void* workspace, size_t workspace_bytes,
                              void* stream) {
  const bool do_rgb = flags & VP_RGB, do_diff = flags & VP_DEPTH_DIFF, need_depth = do_diff || (do_rgb && (flags & VP_RESOLVE));
  GDRN_REQUIRE(inst_off && N > 0 && n >= 0 && H > 0 && W > 0, "vis_poses: need inst_off and N, H, W > 0");
  GDRN_REQUIRE(max_inst >= 0 && max_inst <= VP_MAX_INST, "vis_poses: max_inst (instances of one image) must be <= 3000");
  GDRN_REQUIRE((flags & ~7) == 0 && (do_rgb || do_diff), "vis_poses: flags must select rgb and / or depth_diff");
  GDRN_REQUIRE(!do_rgb || (rgb && ren_rgb && blend && boxes && (n == 0 || m_rgb)),
               "vis_poses: the rgb outputs need m_rgb, rgb, ren_rgb, blend and boxes");
  GDRN_REQUIRE(!need_depth || (ren_depth && (n == 0 || m_depth)), "vis_poses: visibility needs m_depth and ren_depth");
  GDRN_REQUIRE(!do_diff || (depth && diff_vis && diff_minmax && diff_sum && diff_count),
               "vis_poses: depth_diff needs depth and its outputs");
  GDRN_REQUIRE((long long)H * W <= INT_MAX, "vis_poses: image too large");
  GDRN_REQUIRE(workspace && workspace_bytes >= gdrn_vis_poses_workspace_bytes(N, H, W), "vis_poses: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const long long HW = (long long)H * W;
  const int slices = (int)min((HW + VP_THREADS * VP_PIX_PER_THREAD - 1) / (VP_THREADS * VP_PIX_PER_THREAD),
                              (long long)VP_MAX_SLICES);
  uint8_t* ws = (uint8_t*)workspace;
  VisStats* stats = (VisStats*)ws;
  double* sum_part = (double*)(ws + vis_stats_bytes(N));
  float* diff = (float*)(ws + vis_stats_bytes(N) + (size_t)N * VP_MAX_SLICES * 8);
  const int init = max(N, n * 4);
  vis_init_kernel<<<(init + 255) / 256, 256, 0, st>>>(stats, N, do_rgb ? boxes : nullptr, n);
  const size_t smem = do_rgb ? (size_t)max_inst * 16 : 0;
  vis_composite_kernel<<<dim3(slices, N), VP_THREADS, smem, st>>>(m_rgb, m_depth, inst_off, rgb, depth, H, W, flags, ren_rgb,
                                                               ren_depth, blend, boxes, diff, stats, sum_part);
  int launches = 2;
  if (do_diff) {
    vis_diff_range_kernel<<<dim3(slices, N), VP_THREADS, 0, st>>>(diff, H, W, stats, sum_part, diff_minmax, diff_sum,
                                                                  diff_count);
    vis_diff_image_kernel<<<dim3(slices, N), VP_THREADS, 0, st>>>(diff, ren_depth, depth, H, W, stats, diff_vis);
    launches += 2;
  }
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(launches);
  return GDRN_OK;
}

// ---- pose outlines (the per-dataset vis_poses_full scripts) --------------------------------------------------------
namespace {

// mmcv.bgr2gray == cv2.cvtColor(BGR2GRAY) on u8: OpenCV 4's 15-bit fixed-point weights of R 0.299, G 0.587, B 0.114,
// rounded (equal to cv2 on all 2^24 inputs; the older 14-bit weights 4899 / 9617 / 1868 differ on about 0.3 % of them).
// rgb_order: the input's channels are R, G, B (else B, G, R); the output is the same either way.
__global__ void vis_gray3_kernel(const uint8_t* __restrict__ img, long long npx, int rgb_order, uint8_t* __restrict__ out) {
  const int ib = rgb_order ? 2 : 0, ir = 2 - ib;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
    const unsigned b = img[i * 3 + ib], g = img[i * 3 + 1], r = img[i * 3 + ir];
    const uint8_t y = (uint8_t)((3735u * b + 19235u * g + 9798u * r + 16384u) >> 15);
    out[i * 3] = y; out[i * 3 + 1] = y; out[i * 3 + 2] = y;
  }
}

// get_edge(mask, bw) at (y, x) for the coverage plane c: set, with an unset neighbour bw away inside the image
__device__ __forceinline__ bool edge_at(const float* __restrict__ c, int H, int W, int y, int x, int bw) {
  if (c[(long long)y * W + x] == 0.f) return false;
  return (y + bw < H && c[(long long)(y + bw) * W + x] == 0.f) || (y - bw >= 0 && c[(long long)(y - bw) * W + x] == 0.f) ||
         (x + bw < W && c[(long long)y * W + x + bw] == 0.f) || (x - bw >= 0 && c[(long long)y * W + x - bw] == 0.f);
}

// grid (slices, N): one thread per pixel of image j; the estimate edges win over the GT edges, which win over the render
__global__ void __launch_bounds__(VP_THREADS)
vis_outlines_kernel(const float* __restrict__ shaded, const float* __restrict__ cover, const int* __restrict__ inst_off,
                    const uint8_t* __restrict__ is_gt, int H, int W, int bw, uint8_t* __restrict__ out) {
  const int j = blockIdx.y, k0 = inst_off[j], k1 = inst_off[j + 1];
  const long long HW = (long long)H * W;
  for (long long p = (long long)blockIdx.x * VP_THREADS + threadIdx.x; p < HW; p += (long long)gridDim.x * VP_THREADS) {
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    bool est = false, gt = false;
    for (int k = k0; k < k1 && !est; ++k) {
      const bool g = is_gt[k] != 0;
      if (g && gt) continue;
      if (edge_at(cover + (size_t)k * HW, H, W, y, x, bw)) (g ? gt : est) = true;
    }
    const size_t o = ((size_t)j * HW + p) * 3;
    if (est) { out[o] = 0; out[o + 1] = 255; out[o + 2] = 0; continue; }
    if (gt) { out[o] = 255; out[o + 1] = 0; out[o + 2] = 0; continue; }
#pragma unroll
    for (int c = 0; c < 3; ++c)   // image_tensor = bgr(shaded) * 255, then (image_tensor + 0.5).astype(uint8), all f32
      out[o + c] = (uint8_t)__fadd_rn(__fmul_rn(shaded[o + 2 - c], 255.f), 0.5f);
  }
}

}  // namespace

extern "C" int gdrn_vis_gray3(const uint8_t* img, int N, int H, int W, int rgb_order, uint8_t* out, void* stream) {
  GDRN_REQUIRE(img && out && N > 0 && H > 0 && W > 0, "vis_gray3: need img, out and N, H, W > 0");
  const long long npx = (long long)N * H * W;
  const int blocks = (int)min((npx + 255) / 256, 4096LL);
  vis_gray3_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(img, npx, rgb_order, out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_vis_outlines(const float* shaded, const float* cover, const int* inst_off, const uint8_t* is_gt, int N,
                                 int n, int H, int W, int bw, uint8_t* out, void* stream) {
  GDRN_REQUIRE(shaded && inst_off && out && N > 0 && n >= 0 && H > 0 && W > 0, "vis_outlines: need shaded, inst_off, "
               "out and N, H, W > 0");
  GDRN_REQUIRE(n == 0 || (cover && is_gt), "vis_outlines: instances need cover and is_gt");
  GDRN_REQUIRE(bw > 0, "vis_outlines: bw must be > 0");
  GDRN_REQUIRE((long long)H * W <= INT_MAX, "vis_outlines: image too large");
  const long long HW = (long long)H * W;
  const int slices = (int)min((HW + VP_THREADS * VP_PIX_PER_THREAD - 1) / (VP_THREADS * VP_PIX_PER_THREAD),
                              (long long)VP_MAX_SLICES);
  vis_outlines_kernel<<<dim3(slices, N), VP_THREADS, 0, (cudaStream_t)stream>>>(shaded, cover, inst_off, is_gt, H, W, bw,
                                                                                out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
