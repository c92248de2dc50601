// The YOLOX test-time letterbox (det/yolox/data/data_augment.py preproc after base_data_from_list.load_resized_img):
// resize to (int(w * r), int(h * r)) with r = min(th / h, tw / w), place top-left on a 114-filled th x tw canvas, BGR in
// CHW float32.  The resize is bit-exact to cv2.resize(INTER_LINEAR) on uint8 (cv_resize.cuh);
// scale_x = 1 / (dw / W) in float64, as cv::resize derives it from dsize.
// When the second preproc of ValTransform is not the identity for a size, the host side runs the resize twice through
// a uint8 intermediate, as the reference does.
#include "cv_resize.cuh"

namespace {

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
    cvresize::pixel_u8(img, (long long)W * C, H, W, C, x, y, mode, scale_x, scale_y, v);
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
  const int mode = cvresize::resize_mode(H, W, d.h, d.w, scale_x, scale_y);
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
