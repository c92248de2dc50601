// The YOLOX test-time letterbox (det/yolox/data/data_augment.py preproc after base_data_from_list.load_resized_img):
// resize to (int(w * r), int(h * r)) with r = min(th / h, tw / w), place top-left on a 114-filled th x tw canvas, BGR in
// CHW float32.  The resize is bit-exact to cv2.resize(INTER_LINEAR) on uint8 (OpenCV 4.x resize.cpp), which takes one
// of three paths:
//   * identity (dsize == ssize): a copy;
//   * scale exactly 2 in both axes: INTER_LINEAR silently becomes the INTER_AREA fast path, (a + b + c + d + 2) >> 2;
//   * otherwise the generic fixed-point bilinear path: per output column fx = f32((dx + 0.5) * scale_x - 0.5) in float64,
//     sx = floor(fx), fx -= sx; columns left of 0 or at/after the last one are clamped with fx = 0; the weights are
//     round-half-even(f32(1 - fx) * 2048) and round-half-even(fx * 2048) (11-bit).  Rows use the same formula without
//     the clamp of fy; the two source rows are clamped to [0, H - 1] instead.  The horizontal pass sums in int, the
//     vertical one is (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2.
// scale_x = 1 / (dw / W) in float64, as cv::resize derives it from dsize.
// When the second preproc of ValTransform is not the identity for a size, the host side runs the resize twice through
// a uint8 intermediate, as the reference does.
#include "common.cuh"

namespace {

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

// One thread per (image, output pixel) of the destination: f32 CHW canvas (ch x cw, the resized image top-left, 114
// elsewhere) when out_f != nullptr, else the u8 HWC resized image (ch = dh, cw = dw).
__global__ void __launch_bounds__(256)
letterbox_kernel(const uint8_t* __restrict__ src, int N, int H, int W, int C, int dh, int dw, int mode, double scale_x,
                 double scale_y, int ch, int cw, float* __restrict__ out_f, uint8_t* __restrict__ out_u8) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long plane = (long long)ch * cw;
  if (idx >= plane * N) return;
  const int n = (int)(idx / plane);
  const int y = (int)((idx % plane) / cw), x = (int)(idx % cw);
  int v[3] = {114, 114, 114};
  if (x < dw && y < dh) {
    const uint8_t* img = src + (long long)n * H * W * C;
    const long long rowC = (long long)W * C;
    if (mode == kCopy) {
      const uint8_t* p = img + y * rowC + (long long)x * C;
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = p[C == 1 ? 0 : c];
    } else if (mode == kArea2) {
      const uint8_t* p = img + (2LL * y) * rowC + (2LL * x) * C;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int cs = C == 1 ? 0 : c;
        v[c] = (p[cs] + p[C + cs] + p[rowC + cs] + p[rowC + C + cs] + 2) >> 2;
      }
    } else {
      const Tap tx = linear_tap(x, scale_x, W, true), ty = linear_tap(y, scale_y, H, false);
      const uint8_t* r0 = img + ty.i0 * rowC;
      const uint8_t* r1 = img + ty.i1 * rowC;
      const long long c0 = (long long)tx.i0 * C, c1 = (long long)tx.i1 * C;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int cs = C == 1 ? 0 : c;
        const int h0 = r0[c0 + cs] * tx.w0 + r0[c1 + cs] * tx.w1;
        const int h1 = r1[c0 + cs] * tx.w0 + r1[c1 + cs] * tx.w1;
        v[c] = (((ty.w0 * (h0 >> 4)) >> 16) + ((ty.w1 * (h1 >> 4)) >> 16) + 2) >> 2;
      }
    }
  }
  if (out_f != nullptr) {
    float* o = out_f + (long long)n * 3 * plane + (long long)y * cw + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c * plane] = (float)v[c];
  } else {
    uint8_t* o = out_u8 + ((long long)n * plane + (long long)y * cw + x) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)v[c];
  }
}

struct Size2 {
  int h, w;
};

// preproc's resized size: r = min(th / h, tw / w), (int(h * r), int(w * r))
Size2 letterbox_size(int h, int w, int th, int tw) {
  const double rh = (double)th / h, rw = (double)tw / w;
  const double r = rh < rw ? rh : rw;
  return {(int)(h * r), (int)(w * r)};
}

int launch(const uint8_t* src, int N, int H, int W, int C, Size2 d, int ch, int cw, float* out_f, uint8_t* out_u8,
           cudaStream_t stream) {
  const double scale_x = 1.0 / ((double)d.w / W), scale_y = 1.0 / ((double)d.h / H);
  int mode = kLinear;
  if (d.h == H && d.w == W) mode = kCopy;
  else if (scale_x == 2.0 && scale_y == 2.0) mode = kArea2;
  const long long total = (long long)N * ch * cw;
  letterbox_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(src, N, H, W, C, d.h, d.w, mode, scale_x, scale_y,
                                                                        ch, cw, out_f, out_u8);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

}  // namespace

extern "C" size_t yolox_letterbox_workspace_bytes(int N, int H, int W, int th, int tw) {
  if (N <= 0 || H <= 0 || W <= 0 || th <= 0 || tw <= 0) return 0;
  const Size2 d1 = letterbox_size(H, W, th, tw), d2 = letterbox_size(d1.h, d1.w, th, tw);
  if (d2.h == d1.h && d2.w == d1.w) return 0;
  return (size_t)N * d1.h * d1.w * 3;
}

extern "C" int yolox_letterbox(const uint8_t* images, int N, int H, int W, int C, int th, int tw, float* out,
                               void* workspace, size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(N >= 0 && H > 0 && W > 0 && (C == 1 || C == 3) && th > 0 && tw > 0, "yolox_letterbox: bad shape");
  if (N == 0) return GDRN_OK;
  GDRN_REQUIRE(images && out, "yolox_letterbox: null argument");
  const Size2 d1 = letterbox_size(H, W, th, tw);
  GDRN_REQUIRE(d1.h > 0 && d1.w > 0, "yolox_letterbox: the image resizes to an empty one");
  const Size2 d2 = letterbox_size(d1.h, d1.w, th, tw);
  const cudaStream_t s = (cudaStream_t)stream;
  if (d2.h == d1.h && d2.w == d1.w) return launch(images, N, H, W, C, d1, th, tw, out, nullptr, s);
  GDRN_REQUIRE(workspace && workspace_bytes >= yolox_letterbox_workspace_bytes(N, H, W, th, tw),
               "yolox_letterbox: this size resizes twice and needs yolox_letterbox_workspace_bytes of workspace");
  uint8_t* mid = (uint8_t*)workspace;
  const int rc = launch(images, N, H, W, C, d1, d1.h, d1.w, nullptr, mid, s);
  if (rc != GDRN_OK) return rc;
  return launch(mid, N, d1.h, d1.w, 3, d2, th, tw, out, nullptr, s);
}
