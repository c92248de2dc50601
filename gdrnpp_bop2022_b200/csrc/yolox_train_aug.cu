// The YOLOX training image pipeline of the reference's MosaicDetection.__getitem__ (det/yolox/data/datasets/
// mosaicdetection.py) with TrainTransform (det/yolox/data/data_augment.py) for a whole batch, uint8 throughout:
//   yolox_train_resize        cv2.resize(INTER_LINEAR) of many images at once (cv_resize.cuh), each optionally placed
//                             top-left on a 114-filled canvas: load_resized_img, the mosaic tiles' resize and mixup's
//                             letterboxed copy-paste image;
//   yolox_train_mosaic_affine the 2h x 2w mosaic (four tiles at their get_mosaic_coordinate rectangles, 114 elsewhere)
//                             seen through cv2.warpAffine(M, (w, h), borderValue=114), without building the mosaic;
//   yolox_train_mixup         mixup's jitter resize, flip, zero pad and crop of the copy-paste canvas, blended
//                             0.5 a + 0.5 b in float32 and truncated;
//   yolox_train_hsv           augment_hsv: u8 RGB/BGR -> HSV (cv2's integer table path), three per-image LUTs, HSV -> u8
//                             (cv2's float path with FMA and truncation, as cv2 4.x's vector code computes it);
//   yolox_train_preproc       TrainTransform's mirror and preproc letterbox into 114, optionally stored transposed
//                             ((w, h, c), where the wrapper's HSV and colour program run);
//   yolox_train_pack          the finished u8 images, transposed back where needed, as float32 CHW.
// Every random choice arrives from the host in the per-sample record (gdrnpp_bop2022_b200/yolox_train_batch.py); the
// kernels are deterministic functions of (images, record).  No FMA contraction except where cv2 uses one (__fmaf_rn).
#include "crop_common.cuh"
#include "cv_resize.cuh"

namespace {

constexpr int kBorder = 114;
constexpr int kJob = 8;    // resize job: src_off, sh, sw, dst_off, dh, dw, ch, cw
constexpr int kTile = 8;   // mosaic tile: lx1, ly1, lx2, ly2, padw, padh, tile_w, tile_off

__global__ void __launch_bounds__(256)
resize_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const long long* __restrict__ jobs) {
  const long long* j = jobs + (long long)kJob * blockIdx.y;
  const int sh = (int)j[1], sw = (int)j[2], dh = (int)j[4], dw = (int)j[5], ch = (int)j[6], cw = (int)j[7];
  const double scale_x = 1.0 / ((double)dw / sw), scale_y = 1.0 / ((double)dh / sh);
  const int mode = cvresize::resize_mode(sh, sw, dh, dw, scale_x, scale_y);
  const long long plane = (long long)ch * cw;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < plane; p += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(p / cw), x = (int)(p % cw);
    int v[3] = {kBorder, kBorder, kBorder};
    if (x < dw && y < dh) cvresize::pixel_u8(src + j[0], 3LL * sw, sh, sw, 3, x, y, mode, scale_x, scale_y, v);
    uint8_t* o = dst + j[3] + p * 3;
    o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
  }
}

// one pixel of the virtual mosaic: the last pasted tile covering (x, y), else 114
__device__ __forceinline__ const uint8_t* mosaic_px(const uint8_t* __restrict__ tiles, const long long* __restrict__ t, int x, int y) {
  for (int k = 3; k >= 0; --k) {
    const long long* q = t + kTile * k;
    if (x >= q[0] && y >= q[1] && x < q[2] && y < q[3])
      return tiles + q[7] + ((long long)(y - q[5]) * q[6] + (x - q[4])) * 3;
  }
  return nullptr;
}

__global__ void __launch_bounds__(256)
mosaic_affine_kernel(const uint8_t* __restrict__ tiles, const long long* __restrict__ tile_info, const double* __restrict__ M,
                     const int* __restrict__ sel, int n_sel, int oh, int ow, uint8_t* __restrict__ out) {
  const long long plane = (long long)oh * ow;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= plane * n_sel) return;
  const int i = (int)(idx / plane);
  const int y = (int)((idx % plane) / ow), x = (int)(idx % ow);
  const long long* t = tile_info + 4LL * kTile * i;
  double iM[6];
  crop::invert_affine(M + 6LL * i, iM);
  const crop::U8Tap tap = crop::u8_tap(crop::src_coord(iM, x, y, false), 2 * oh, 2 * ow);
  int v[3] = {kBorder, kBorder, kBorder};
  // OpenCV's BORDER_CONSTANT: a tap outside the 2h x 2w source reads the border value; a fully outside position is it
  if (tap.in[0] || tap.in[1] || tap.in[2] || tap.in[3]) {
    const uint8_t* p[4];
    for (int k = 0; k < 4; ++k) p[k] = tap.in[k] ? mosaic_px(tiles, t, tap.sx + (k & 1), tap.sy + (k >> 1)) : nullptr;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int s = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) s += (p[k] ? p[k][c] : kBorder) * tap.w[k];
      v[c] = crop::u8_round(s);
    }
  }
  uint8_t* o = out + ((long long)sel[i] * plane + (long long)y * ow + x) * 3;
  o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
}

// mp per selected sample: canvas_off, jit_h, jit_w, flip, x_offset, y_offset
__global__ void __launch_bounds__(256)
mixup_kernel(uint8_t* __restrict__ img, const uint8_t* __restrict__ canvases, const long long* __restrict__ mp,
             const int* __restrict__ sel, int n_sel, int oh, int ow) {
  const long long plane = (long long)oh * ow;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= plane * n_sel) return;
  const int i = (int)(idx / plane);
  const int y = (int)((idx % plane) / ow), x = (int)(idx % ow);
  const long long* m = mp + 6LL * i;
  const int dh = (int)m[1], dw = (int)m[2];
  const int X = x + (int)m[4], Y = y + (int)m[5];
  int b[3] = {0, 0, 0};   // padded_img is zeros outside the jittered canvas
  if (X < dw && Y < dh) {
    const double scale_x = 1.0 / ((double)dw / ow), scale_y = 1.0 / ((double)dh / oh);
    const int mode = cvresize::resize_mode(oh, ow, dh, dw, scale_x, scale_y);
    cvresize::pixel_u8(canvases + m[0], 3LL * ow, oh, ow, 3, m[3] ? dw - 1 - X : X, Y, mode, scale_x, scale_y, b);
  }
  uint8_t* o = img + ((long long)sel[i] * plane + (long long)y * ow + x) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = (uint8_t)(int)__fadd_rn(__fmul_rn(0.5f, (float)o[c]), __fmul_rn(0.5f, (float)b[c]));
}

// cv2 RGB2HSV_b tables: (255 << 12) / v and (180 << 12) / (6 diff), rounded half to even
__device__ __forceinline__ int sdiv(int v) { return v ? __double2int_rn(__ddiv_rn((double)(255 << 12), (double)v)) : 0; }
__device__ __forceinline__ int hdiv(int d) { return d ? __double2int_rn(__ddiv_rn((double)(180 << 12), __dmul_rn(6.0, (double)d))) : 0; }

__device__ __forceinline__ int trunc_u8(float x) {
  const float t = __fmul_rn(x, 255.f);
  return t <= 0.f ? 0 : (t >= 255.f ? 255 : (int)t);
}

// HSV -> RGB: which of (v, v(1 - s), v(1 - s f), v(1 - s(1 - f))) each of b, g, r takes per sector, 4 bits per channel
__constant__ int kSector[6] = {0x031, 0x201, 0x103, 0x120, 0x310, 0x012};

// entries: off (into pool), npix; lut per entry [3][256]; rgb: channel 0 is R (else B)
__global__ void __launch_bounds__(256)
hsv_kernel(uint8_t* __restrict__ pool, const long long* __restrict__ ent, const uint8_t* __restrict__ lut, int rgb) {
  const long long* e = ent + 2LL * blockIdx.y;
  const uint8_t* L = lut + 768LL * blockIdx.y;
  const int ri = rgb ? 0 : 2, bi = 2 - ri;
  const float inv255 = __fdiv_rn(1.f, 255.f), hscale = __fdiv_rn(6.f, 180.f);
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < e[1]; p += (long long)gridDim.x * blockDim.x) {
    uint8_t* q = pool + e[0] + p * 3;
    const int r = q[ri], g = q[1], b = q[bi];
    const int v = max(max(b, g), r), vmin = min(min(b, g), r), diff = v - vmin;
    const int s = (diff * sdiv(v) + (1 << 11)) >> 12;
    int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
    h = (h * hdiv(diff) + (1 << 11)) >> 12;
    if (h < 0) h += 180;
    const int H = L[h], S = L[256 + s], V = L[512 + v];
    int o[3];   // b, g, r
    if (S == 0) {
      o[0] = o[1] = o[2] = V;
    } else {
      const float vf = __fmul_rn((float)V, inv255), sf = __fmul_rn((float)S, inv255);
      float hf = __fmul_rn((float)H, hscale);
      int sector = (int)floorf(hf);
      hf = __fsub_rn(hf, (float)sector);
      if ((unsigned)sector >= 6u) { sector = 0; hf = 0.f; }
      const float t1 = __fmul_rn(vf, __fsub_rn(1.f, sf)), t2 = __fmul_rn(vf, __fmaf_rn(-sf, hf, 1.f));
      const float t3 = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.f, hf), 1.f));
#pragma unroll
      for (int c = 0; c < 3; ++c) {   // cv2's sector_data {{1,3,0}, {1,0,2}, {3,0,1}, {0,2,1}, {0,1,3}, {2,1,0}}
        const int k = (kSector[sector] >> (4 * c)) & 3;
        o[c] = trunc_u8(k == 0 ? vf : (k == 1 ? t1 : (k == 2 ? t2 : t3)));
      }
    }
    q[bi] = (uint8_t)o[0]; q[1] = (uint8_t)o[1]; q[ri] = (uint8_t)o[2];
  }
}

// info per sample: src_off, sh, sw, flip, transpose.  preproc: resize to (int(sh r), int(sw r)), r = min(oh / sh, ow / sw)
__global__ void __launch_bounds__(256)
preproc_kernel(const uint8_t* __restrict__ pool, const long long* __restrict__ info, int oh, int ow, uint8_t* __restrict__ out) {
  const int b = blockIdx.y;
  const long long* f = info + 5LL * b;
  const int sh = (int)f[1], sw = (int)f[2];
  const double r = fmin((double)oh / sh, (double)ow / sw);
  const int dh = (int)(sh * r), dw = (int)(sw * r);
  const double scale_x = 1.0 / ((double)dw / sw), scale_y = 1.0 / ((double)dh / sh);
  const int mode = cvresize::resize_mode(sh, sw, dh, dw, scale_x, scale_y);
  const long long plane = (long long)oh * ow;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < plane; p += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(p / ow), x = (int)(p % ow);
    int v[3] = {kBorder, kBorder, kBorder};
    if (x < dw && y < dh) cvresize::pixel_u8(pool + f[0], 3LL * sw, sh, sw, 3, x, y, mode, scale_x, scale_y, v, f[3] != 0);
    uint8_t* o = out + (b * plane + (f[4] ? (long long)x * oh + y : p)) * 3;
    o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
  }
}

__global__ void __launch_bounds__(256)
pack_kernel(const uint8_t* __restrict__ img, const int* __restrict__ transposed, int n, int oh, int ow, float* __restrict__ out) {
  const long long plane = (long long)oh * ow;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= plane * n) return;
  const int b = (int)(idx / plane);
  const int y = (int)((idx % plane) / ow), x = (int)(idx % ow);
  const uint8_t* q = img + (b * plane + (transposed[b] ? (long long)x * oh + y : (long long)y * ow + x)) * 3;
  float* o = out + (long long)b * 3 * plane + (long long)y * ow + x;
  o[0] = (float)q[0]; o[plane] = (float)q[1]; o[2 * plane] = (float)q[2];
}

unsigned grid_x(long long work) { return (unsigned)min((work + 255) / 256, 1024LL); }

}  // namespace

extern "C" int yolox_train_resize(const uint8_t* src, uint8_t* dst, const long long* jobs, int n_jobs, long long max_plane,
                                  void* stream) {
  GDRN_REQUIRE(n_jobs >= 0 && max_plane >= 0, "yolox_train_resize: bad shape");
  if (n_jobs == 0) return GDRN_OK;
  GDRN_REQUIRE(src && dst && jobs && src != dst, "yolox_train_resize: null argument");
  resize_kernel<<<dim3(grid_x(max_plane), n_jobs), 256, 0, (cudaStream_t)stream>>>(src, dst, jobs);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int yolox_train_mosaic_affine(const uint8_t* tiles, const long long* tile_info, const double* M, const int* sel,
                                         int n_sel, int oh, int ow, uint8_t* out, void* stream) {
  GDRN_REQUIRE(n_sel >= 0 && oh > 0 && ow > 0, "yolox_train_mosaic_affine: bad shape");
  if (n_sel == 0) return GDRN_OK;
  GDRN_REQUIRE(tiles && tile_info && M && sel && out, "yolox_train_mosaic_affine: null argument");
  const long long total = (long long)n_sel * oh * ow;
  mosaic_affine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tiles, tile_info, M, sel, n_sel, oh,
                                                                                          ow, out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int yolox_train_mixup(uint8_t* images, const uint8_t* canvases, const long long* params, const int* sel, int n_sel,
                                 int oh, int ow, void* stream) {
  GDRN_REQUIRE(n_sel >= 0 && oh > 0 && ow > 0, "yolox_train_mixup: bad shape");
  if (n_sel == 0) return GDRN_OK;
  GDRN_REQUIRE(images && canvases && params && sel, "yolox_train_mixup: null argument");
  const long long total = (long long)n_sel * oh * ow;
  mixup_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(images, canvases, params, sel, n_sel, oh, ow);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int yolox_train_hsv(uint8_t* pool, const long long* entries, const uint8_t* luts, int n, long long max_pix, int rgb,
                               void* stream) {
  GDRN_REQUIRE(n >= 0 && max_pix >= 0, "yolox_train_hsv: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(pool && entries && luts, "yolox_train_hsv: null argument");
  hsv_kernel<<<dim3(grid_x(max_pix), n), 256, 0, (cudaStream_t)stream>>>(pool, entries, luts, rgb);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int yolox_train_preproc(const uint8_t* pool, const long long* info, int n, int oh, int ow, uint8_t* out,
                                   void* stream) {
  GDRN_REQUIRE(n >= 0 && oh > 0 && ow > 0, "yolox_train_preproc: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(pool && info && out, "yolox_train_preproc: null argument");
  preproc_kernel<<<dim3(grid_x((long long)oh * ow), n), 256, 0, (cudaStream_t)stream>>>(pool, info, oh, ow, out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int yolox_train_pack(const uint8_t* images, const int* transposed, int n, int oh, int ow, float* out, void* stream) {
  GDRN_REQUIRE(n >= 0 && oh > 0 && ow > 0, "yolox_train_pack: bad shape");
  if (n == 0) return GDRN_OK;
  GDRN_REQUIRE(images && transposed && out, "yolox_train_pack: null argument");
  const long long total = (long long)n * oh * ow;
  pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(images, transposed, n, oh, ow, out);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
