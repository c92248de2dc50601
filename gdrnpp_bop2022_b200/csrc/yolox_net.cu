// YOLOX detector network (det/yolox/models: CSPDarknet + YOLOPAFPN + YOLOXHead, inference) on the GPU (sm_90a).
//
// Every convolution of the network is a dense conv + folded BatchNorm + SiLU (BaseConv), or a plain conv with a bias
// (the head's prediction convs).  yolox_conv runs one as an implicit GEMM on the tensor cores:
//   out[m, co_off + n] = act(sum_k A[m, k] * W[n, k] + bias[n]) (+ resid[m, cr_off + n])
// m = flat NHWC output pixel (b, oy, ox), k = (ky, kx, ci).  Activations are fp32 NHWC buffers addressed by a channel
// offset and a pixel stride, so a conv reads or writes one channel slice of a wider buffer and the torch.cat of
// CSPLayer / SPPBottleneck / YOLOPAFPN costs nothing.  Tiles run over the flat pixel index, so any map size works and
// only the last 128-row tile of a layer is partial.
// Precision: split = 1 (bf16x3) forms A = A_hi + A_lo, W = W_hi + W_lo in bf16 and sums A_lo*W_hi + A_hi*W_lo + A_hi*W_hi
// in fp32 (about 16 mantissa bits per product); split = 0 (bf16) keeps A_hi*W_hi only.
//
// Launched through gdrn_launch_dep (PDL), so every kernel below starts with griddep_launch / griddep_wait.
// Small kernels around it: Focus (space-to-depth of the [B,3,H,W] input), SPP max-pools, nearest x2 upsample into a
// concat slice, the head output assembly (decode + sigmoid into det_preds [B, A, 5 + nc]) and the keep-single-instance
// post-process of the reference predictor (core/gdrn_modeling/demo/predictor_yolo.py:84-140).
#include "common.cuh"

namespace {

constexpr int CV_BM = 128, CV_BN = 64, CV_BK = 32;
constexpr int CV_PITCH = CV_BK + 8;   // bf16 elements per shared-memory row: 80 B, fragment loads are conflict-free
constexpr int CV_THREADS = 256;

struct ConvArgs {
  const float* x; int ldx, cx_off, Cin, H, W;
  const __nv_bfloat16* w_hi; const __nv_bfloat16* w_lo; int K;   // W [>= Cout rows][K], K = ks * ks * Cin
  const float* bias; int Cout;
  int ks, stride, pad, OH, OW; long long M;
  float* out; int ldo, co_off;
  const float* resid; int ldr, cr_off;
  int act;
};

__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 128 x 64 output tile per CTA, 8 warps of 32 x 32; the next k-chunk is fetched into registers while the tensor cores run
// the current one.
template <bool SPLIT>
__global__ void __launch_bounds__(CV_THREADS) yolox_conv_kernel(const ConvArgs p) {
  ptx::griddep_launch();
  ptx::griddep_wait();   // PDL: the producer kernel's writes are visible from here on
  __shared__ __align__(16) __nv_bfloat16 sa[SPLIT ? 2 : 1][CV_BM][CV_PITCH];
  __shared__ __align__(16) __nv_bfloat16 sb[SPLIT ? 2 : 1][CV_BN][CV_PITCH];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 3, wn = warp >> 2;
  const long long m0 = (long long)blockIdx.x * CV_BM;
  const int n0 = blockIdx.y * CV_BN;

  // A loader: rows tid/4 and tid/4 + 64, 8 channels (one tap) at column (tid & 3) * 8 of the chunk
  const int lg = tid & 3;
  int a_b[2], a_iy[2], a_ix[2];
  bool a_ok[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long m = m0 + (tid >> 2) + 64 * r;
    a_ok[r] = m < p.M;
    const long long mm = a_ok[r] ? m : 0;
    const int ox = (int)(mm % p.OW);
    const long long t = mm / p.OW;
    a_iy[r] = (int)(t % p.OH) * p.stride - p.pad;
    a_ix[r] = ox * p.stride - p.pad;
    a_b[r] = (int)(t / p.OH);
  }
  // W loader: row tid/4, 8 k at (tid & 3) * 8
  const int b_row = n0 + (tid >> 2);
  const bool b_ok = b_row < p.Cout;

  float4 ra[2][2];
  uint4 rb[2];
  auto fetch = [&](int k0) {
    const int k = k0 + lg * 8;
    const bool kin = k < p.K;
    const int tap = kin ? k / p.Cin : 0;
    const int ci = k - tap * p.Cin;
    const int ky = tap / p.ks, kx = tap - ky * p.ks;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int iy = a_iy[r] + ky, ix = a_ix[r] + kx;
      if (kin && a_ok[r] && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
        const float4* src = reinterpret_cast<const float4*>(
            p.x + ((long long)(a_b[r] * p.H + iy) * p.W + ix) * p.ldx + p.cx_off + ci);
        ra[r][0] = __ldg(src);
        ra[r][1] = __ldg(src + 1);
      } else {
        ra[r][0] = ra[r][1] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    const bool wk = kin && b_ok;
    rb[0] = wk ? __ldg(reinterpret_cast<const uint4*>(p.w_hi + (long long)b_row * p.K + k)) : make_uint4(0, 0, 0, 0);
    if constexpr (SPLIT) rb[1] = wk ? __ldg(reinterpret_cast<const uint4*>(p.w_lo + (long long)b_row * p.K + k)) : make_uint4(0, 0, 0, 0);
  };
  auto stash = [&]() {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float v[8] = {ra[r][0].x, ra[r][0].y, ra[r][0].z, ra[r][0].w, ra[r][1].x, ra[r][1].y, ra[r][1].z, ra[r][1].w};
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
        hi[j] = *reinterpret_cast<const uint32_t*>(&h);
        if constexpr (SPLIT) {
          const __nv_bfloat162 l = __floats2bfloat162_rn(v[2 * j] - __low2float(h), v[2 * j + 1] - __high2float(h));
          lo[j] = *reinterpret_cast<const uint32_t*>(&l);
        }
      }
      const int row = (tid >> 2) + 64 * r;
      *reinterpret_cast<uint4*>(&sa[0][row][lg * 8]) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      if constexpr (SPLIT) *reinterpret_cast<uint4*>(&sa[1][row][lg * 8]) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
    *reinterpret_cast<uint4*>(&sb[0][tid >> 2][lg * 8]) = rb[0];
    if constexpr (SPLIT) *reinterpret_cast<uint4*>(&sb[1][tid >> 2][lg * 8]) = rb[1];
  };

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

  const int g = lane >> 2, t = lane & 3;
  fetch(0);
  for (int k0 = 0; k0 < p.K; k0 += CV_BK) {
    __syncthreads();   // the previous chunk's fragments have been read
    stash();
    __syncthreads();
    if (k0 + CV_BK < p.K) fetch(k0 + CV_BK);
#pragma unroll
    for (int kk = 0; kk < CV_BK; kk += 16) {
      uint32_t af[SPLIT ? 2 : 1][2][4], bf[SPLIT ? 2 : 1][4][2];
#pragma unroll
      for (int h = 0; h < (SPLIT ? 2 : 1); ++h) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = wm * 32 + i * 16 + g;
          af[h][i][0] = *reinterpret_cast<const uint32_t*>(&sa[h][r][kk + 2 * t]);
          af[h][i][1] = *reinterpret_cast<const uint32_t*>(&sa[h][r + 8][kk + 2 * t]);
          af[h][i][2] = *reinterpret_cast<const uint32_t*>(&sa[h][r][kk + 8 + 2 * t]);
          af[h][i][3] = *reinterpret_cast<const uint32_t*>(&sa[h][r + 8][kk + 8 + 2 * t]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = wn * 32 + j * 8 + g;
          bf[h][j][0] = *reinterpret_cast<const uint32_t*>(&sb[h][c][kk + 2 * t]);
          bf[h][j][1] = *reinterpret_cast<const uint32_t*>(&sb[h][c][kk + 8 + 2 * t]);
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if constexpr (SPLIT) {   // small terms first
            mma_bf16(acc[i][j], af[1][i], bf[0][j][0], bf[0][j][1]);
            mma_bf16(acc[i][j], af[0][i], bf[1][j][0], bf[1][j][1]);
          }
          mma_bf16(acc[i][j], af[0][i], bf[0][j][0], bf[0][j][1]);
        }
    }
  }

  // epilogue: bias, SiLU, shortcut add after the activation (Bottleneck.use_add), store into the output slice
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int n = n0 + wn * 32 + j * 8 + 2 * t;
    const float b0 = (p.bias && n < p.Cout) ? __ldg(p.bias + n) : 0.f;
    const float b1 = (p.bias && n + 1 < p.Cout) ? __ldg(p.bias + n + 1) : 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long m = m0 + wm * 32 + i * 16 + g + 8 * h;
        if (m >= p.M) continue;
        float v[2] = {acc[i][j][2 * h] + b0, acc[i][j][2 * h + 1] + b1};
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (n + e >= p.Cout) continue;
          float y = v[e];
          if (p.act) y = __fdividef(y, 1.f + __expf(-y));
          if (p.resid) y += p.resid[m * p.ldr + p.cr_off + n + e];
          p.out[m * p.ldo + p.co_off + n + e] = y;
        }
      }
  }
}

// Focus (network_blocks.py:181-196): [B,3,H,W] -> NHWC [B,H/2,W/2,16], channels (TL, BL, TR, BR) x 3, 12..15 zero
__global__ void yolox_focus_kernel(const float* __restrict__ img, int B, int H, int W, float* __restrict__ out) {
  ptx::griddep_launch();
  ptx::griddep_wait();   // PDL: the producer kernel's writes are visible from here on
  const int h2 = H / 2, w2 = W / 2;
  const long long n = (long long)B * h2 * w2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % w2);
  const long long tt = i / w2;
  const int y = (int)(tt % h2), b = (int)(tt / h2);
  float v[16];
  const int dy[4] = {0, 1, 0, 1}, dx[4] = {0, 0, 1, 1};
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      v[q * 3 + c] = __ldg(img + (((long long)b * 3 + c) * H + 2 * y + dy[q]) * W + 2 * x + dx[q]);
  v[12] = v[13] = v[14] = v[15] = 0.f;
  float4* o = reinterpret_cast<float4*>(out + i * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q) o[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
}

// one axis of torch's upsample_bilinear2d (align_corners=False, output size given): source row / column i0, the step to
// the next one (0 at the last) and the weight of the next one; scale = (float)in / out
struct YSample { int i0, step; float lam; };
__device__ __forceinline__ YSample yolox_bilinear_axis(int dst, float scale, int in) {
  float src = scale * (dst + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  YSample s;
  s.i0 = (int)src;
  s.step = s.i0 < in - 1 ? 1 : 0;
  s.lam = src - (float)s.i0;
  return s;
}

// Focus of the multi-scale test input (model_utils.scale_img: bilinear resize of [B,3,H,W] to the content size sh x sw,
// then padding right / bottom with 0.447 * 255 up to PH x PW) without materialising the scaled image: every pixel Focus
// reads is sampled from the original input.  Output as yolox_focus_kernel: NHWC [B,PH/2,PW/2,16], (TL, BL, TR, BR) x 3.
__global__ void yolox_focus_resample_kernel(const float* __restrict__ img, int B, int H, int W, int PH, int PW, int sh, int sw,
                                            float scale_h, float scale_w, float* __restrict__ out) {
  ptx::griddep_launch();
  ptx::griddep_wait();   // PDL: the producer kernel's writes are visible from here on
  const int h2 = PH / 2, w2 = PW / 2;
  const long long n = (long long)B * h2 * w2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % w2);
  const long long tt = i / w2;
  const int y = (int)(tt % h2), b = (int)(tt / h2);
  const float pad = (float)(0.447 * 255);
  YSample ry[2], rx[2];
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    ry[d] = yolox_bilinear_axis(2 * y + d, scale_h, H);
    rx[d] = yolox_bilinear_axis(2 * x + d, scale_w, W);
  }
  float v[16];
  const int dy[4] = {0, 1, 0, 1}, dx[4] = {0, 0, 1, 1};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const YSample& sy = ry[dy[q]];
    const YSample& sx = rx[dx[q]];
    const bool inside = 2 * y + dy[q] < sh && 2 * x + dx[q] < sw;
    const float h1l = sy.lam, h0l = 1.f - h1l, w1l = sx.lam, w0l = 1.f - w1l;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float r = pad;
      if (inside) {
        const float* p0 = img + (((long long)b * 3 + c) * H + sy.i0) * W + sx.i0;
        const float* p1 = p0 + (long long)sy.step * W;
        r = h0l * (w0l * __ldg(p0) + w1l * __ldg(p0 + sx.step)) + h1l * (w0l * __ldg(p1) + w1l * __ldg(p1 + sx.step));
      }
      v[q * 3 + c] = r;
    }
  }
  v[12] = v[13] = v[14] = v[15] = 0.f;
  float4* o = reinterpret_cast<float4*>(out + i * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q) o[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
}

// SPPBottleneck (network_blocks.py:118-133): max-pools 5 / 9 / 13, stride 1, padding k/2 (-inf, like nn.MaxPool2d) of the
// C channels at slice 0 of buf, written to slices C, 2C, 3C of the same buffer
__global__ void yolox_spp_kernel(float* __restrict__ buf, int B, int H, int W, int ld, int C) {
  ptx::griddep_launch();
  ptx::griddep_wait();   // PDL: the producer kernel's writes are visible from here on
  const long long n = (long long)B * H * W * C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const long long pix = i / C;
  const int x = (int)(pix % W);
  const long long tt = pix / W;
  const int y = (int)(tt % H), b = (int)(tt / H);
  float m5 = -INFINITY, m9 = -INFINITY, m13 = -INFINITY;
  for (int dy = -6; dy <= 6; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -6; dx <= 6; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      const float v = buf[(((long long)b * H + yy) * W + xx) * ld + c];
      const int r = max(abs(dy), abs(dx));
      m13 = fmaxf(m13, v);
      if (r <= 4) m9 = fmaxf(m9, v);
      if (r <= 2) m5 = fmaxf(m5, v);
    }
  }
  float* o = buf + pix * ld + c;
  o[C] = m5;
  o[2 * C] = m9;
  o[3 * C] = m13;
}

// nearest x2 upsample (yolo_pafpn.py:90-97) of C channels [B,h,w] at src slice -> [B,2h,2w] at dst slice
__global__ void yolox_upsample2x_kernel(const float* __restrict__ src, int lds, int so, float* __restrict__ dst, int ldd, int dof,
                                        int B, int h, int w, int C) {
  ptx::griddep_launch();
  ptx::griddep_wait();   // PDL: the producer kernel's writes are visible from here on
  const long long n = (long long)B * 4 * h * w * C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const long long pix = i / C;
  const int x = (int)(pix % (2 * w));
  const long long tt = pix / (2 * w);
  const int y = (int)(tt % (2 * h)), b = (int)(tt / (2 * h));
  dst[pix * ldd + dof + c] = __ldg(src + (((long long)b * h + y / 2) * w + x / 2) * lds + so + c);
}

// head output of one level (yolo_head.py:191-254): raw [B, h*w, 5 + nc] (reg 4 | obj | cls) -> det_preds rows
// [a_off, a_off + h*w) of [B, A, 5 + nc]: xy = (xy + grid) * stride, wh = exp(wh) * stride, sigmoid(obj), sigmoid(cls).
// The four box columns are then multiplied by inv_scale: the test-time-augmentation de-scale det[..., :4] /= s, which
// torch evaluates on CUDA for a Python-scalar divisor as x * (1.0f / (float)s).  inv_scale = 1 leaves them exact.
__global__ void yolox_head_out_kernel(const float* __restrict__ raw, int B, int h, int w, int nc, int stride, int A, int a_off,
                                      float inv_scale, float* __restrict__ det) {
  ptx::griddep_launch();
  ptx::griddep_wait();   // PDL: the producer kernel's writes are visible from here on
  const int C = 5 + nc;
  const long long n = (long long)B * h * w * C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const long long pix = i / C;
  const int loc = (int)(pix % (h * w)), b = (int)(pix / (h * w));
  const float v = raw[i];
  const float st = (float)stride;
  float o;
  if (c == 0) o = __fmul_rn(__fadd_rn(v, (float)(loc % w)), st);
  else if (c == 1) o = __fmul_rn(__fadd_rn(v, (float)(loc / w)), st);
  else if (c < 4) o = __fmul_rn(expf(v), st);
  else o = __frcp_rn(__fadd_rn(1.f, expf(-v)));
  if (c < 4) o = __fmul_rn(o, inv_scale);
  det[((long long)b * A + a_off + loc) * C + c] = o;
}

// ---- keep-single-instance post-process (predictor_yolo.py:84-140 with keep_single_instance=True, class_agnostic=True) ----
// The reference scores and filters on the device (torch compares the CUDA tensor with conf_thre rounded to fp32), copies
// the selected rows into a host tensor (instance_detections = torch.rand(num_classes, 7)) and so runs torchvision's CPU
// nms: every product rounded on its own and the fp32 IoU compared with the threshold as a double.
// per anchor: class_conf / class_pred = first max over the class scores, score = obj * class_conf
__global__ void yolox_ksi_score_kernel(const float* __restrict__ preds, int B, int A, int nc, float* __restrict__ score,
                                       int* __restrict__ cls) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * A) return;
  const float* P = preds + i * (5 + nc);
  float best = -INFINITY;
  int bc = 0;
  for (int c = 0; c < nc; ++c) {
    const float v = P[5 + c];
    if (v > best) { best = v; bc = c; }
  }
  score[i] = __fmul_rn(P[4], best);
  cls[i] = bc;
}

// per (class, image): the first anchor (lowest index) of the highest conf-passing score of that class; the reference
// starts from max_conf = 0 and replaces on a strictly greater score
__global__ void __launch_bounds__(256) yolox_ksi_select_kernel(const float* __restrict__ score, const int* __restrict__ cls, int A,
                                                               int nc, float conf_thre, int* __restrict__ sel) {
  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  float best = 0.f;
  int bi = -1;
  for (int a = tid; a < A; a += blockDim.x) {
    const float s = score[(long long)b * A + a];
    if (cls[(long long)b * A + a] == c && s >= conf_thre && s > best) { best = s; bi = a; }
  }
  __shared__ float ss[256];
  __shared__ int si[256];
  ss[tid] = best; si[tid] = bi;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) {
      const float s2 = ss[tid + o];
      const int i2 = si[tid + o];
      if (i2 >= 0 && (si[tid] < 0 || s2 > ss[tid] || (s2 == ss[tid] && i2 < si[tid]))) { ss[tid] = s2; si[tid] = i2; }
    }
    __syncthreads();
  }
  if (tid == 0) sel[b * nc + c] = si[0];
}

constexpr int KSI_MAX_CLASSES = 1024;

__device__ __forceinline__ float ksi_iou(const float* a, const float* b) {   // torchvision's CPU nms: (Sa + Sb) - inter
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float width = fmaxf(__fsub_rn(right, left), 0.f), height = fmaxf(__fsub_rn(bottom, top), 0.f);
  const float inter = __fmul_rn(width, height);
  const float Sa = __fmul_rn(__fsub_rn(a[2], a[0]), __fsub_rn(a[3], a[1]));
  const float Sb = __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(Sa, Sb), inter));
}

// one thread per image: the (at most nc) selected rows, class-agnostic greedy NMS in descending score order, kept rows
// written in ascending class order
__global__ void yolox_ksi_nms_kernel(const float* __restrict__ preds, const int* __restrict__ sel, const float* __restrict__ score,
                                     int A, int nc, double nms_thre, float* __restrict__ dets, int* __restrict__ n_det) {
  const int b = blockIdx.x;
  int n_in = 0;
  // sorted insertion by (score desc, class asc) into the output area itself: rows are 7 floats, class kept in row[6]
  float* out = dets + (size_t)b * nc * 7;
  for (int c = 0; c < nc; ++c) {
    const int a = sel[b * nc + c];
    if (a < 0) continue;
    const float* P = preds + ((size_t)b * A + a) * (5 + nc);
    const float cx = P[0], cy = P[1], w = P[2], h = P[3];
    const float hw2 = __fdiv_rn(w, 2.f), hh2 = __fdiv_rn(h, 2.f);
    const float row[7] = {__fsub_rn(cx, hw2), __fsub_rn(cy, hh2), __fadd_rn(cx, hw2), __fadd_rn(cy, hh2), P[4], P[5 + c], (float)c};
    const float s = score[(size_t)b * A + a];
    int pos = n_in;
    while (pos > 0 && __fmul_rn(out[(pos - 1) * 7 + 4], out[(pos - 1) * 7 + 5]) < s) {
      for (int k = 0; k < 7; ++k) out[pos * 7 + k] = out[(pos - 1) * 7 + k];
      --pos;
    }
    for (int k = 0; k < 7; ++k) out[pos * 7 + k] = row[k];
    ++n_in;
  }
  // greedy suppression: a kept row removes every later row with (double)IoU > nms_thre; removed rows get class -1
  for (int i = 0; i < n_in; ++i) {
    if (out[i * 7 + 6] < 0.f) continue;
    for (int j = i + 1; j < n_in; ++j)
      if (out[j * 7 + 6] >= 0.f && (double)ksi_iou(out + i * 7, out + j * 7) > nms_thre) out[j * 7 + 6] = -1.f;
  }
  // compact in ascending class order (selection sort over the survivors: at most nc rows)
  int kept = 0;
  for (int c = 0; c < nc; ++c) {
    for (int i = kept; i < n_in; ++i) {
      if (out[i * 7 + 6] == (float)c) {
        for (int k = 0; k < 7; ++k) { const float tmp = out[kept * 7 + k]; out[kept * 7 + k] = out[i * 7 + k]; out[i * 7 + k] = tmp; }
        ++kept;
        break;
      }
    }
  }
  n_det[b] = kept;
}

inline int blocks_for(long long n, int t) { return (int)((n + t - 1) / t); }

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// YoloxModel: the whole YOLOX forward (CSPDarknet + YOLOPAFPN + YOLOXHead, decode_in_inference) for one
// (depth, width, num_classes, max_batch, H, W, precision).  Weights arrive by reference state-dict name (unfused conv +
// BatchNorm, or fused conv + bias); BatchNorm is folded on the host in float64 once every tensor of a conv is present.
// Activations live in the caller's workspace as fp32 NHWC buffers; a concatenation is one buffer whose producers write
// their own channel slices.  The forward allocates nothing, does not synchronise and launches with PDL.
// Multi-scale test-time augmentation adds one layer plan per scale over the same packed weights (yolox_model_set_scales);
// a scaled plan's Focus step resamples the original input and its head outputs land at the scale's anchor base.
// ---------------------------------------------------------------------------------------------------------------------
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace {

struct YConv {
  int cin = 0, cout = 0, k = 1;
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  float* bias = nullptr;
  bool packed = false;
};

enum { YS_CONV, YS_FOCUS, YS_SPP, YS_UP, YS_HEAD };
struct YStep {
  int kind;
  std::string w;                 // YS_CONV: packed weight name
  int src = -1, s_off = 0, s_c = 0, dst = -1, d_off = 0, d_c = 0, res = -1, r_off = 0;
  int h = 0, wd = 0, ks = 1, stride = 1, act = 1, extra = 0;   // input map size; YS_HEAD: extra = stride, d_off = anchor offset
};
struct YBuf { long long pix; int ld; };   // pixels per image, channels

// the layer plan of one network input size.  Plan 0 runs the create-time H x W input as it is; a test-time-augmentation
// plan runs the input resampled to sh x sw and padded to H x W (model_utils.scale_img) and de-scales its boxes.
struct YPlan {
  int H = 0, W = 0;          // network input size (multiples of 32)
  int sh = 0, sw = 0;        // content size of the resampled image
  bool resample = false;
  float inv_scale = 1.f;     // box de-scale factor 1.0f / (float)s
  int A = 0;                 // anchors
  std::vector<YBuf> bufs;
  std::vector<YStep> steps;
  std::vector<size_t> offs;  // per-buffer workspace offsets (recomputed per chunk size)
};

}  // namespace

struct YoloxModel {
  int nc, max_batch, H, W, split;
  double depth, width;
  std::map<std::string, std::vector<double>> host;   // loaded tensors (float64)
  std::map<std::string, YConv> convs;                  // packed GEMM operands by conv name, shared by every plan
  std::map<std::string, std::vector<std::string>> sources;   // conv name -> the base convs / pred convs it packs from
  std::vector<YPlan> plans;                            // [0]: the create-time size; then one per non-unit TTA scale
  std::vector<int> tta_plan;                           // yolox_model_set_scales: plan index per scale, in scale order
  int A_tta = 0;                                       // anchors summed over the scales
};

namespace {

size_t yx_align(size_t v) { return (v + 255) & ~(size_t)255; }

int yx_buf(YPlan* pl, int h, int w, int c) { pl->bufs.push_back({(long long)h * w, c}); return (int)pl->bufs.size() - 1; }

// conv shapes do not depend on the input size: the first plan declares them, later plans find them declared
void yx_conv_decl(YoloxModel* m, const std::string& name, int cin, int cout, int k, const std::vector<std::string>& src) {
  if (m->convs.count(name)) return;
  YConv c; c.cin = cin; c.cout = cout; c.k = k;
  m->convs[name] = c;
  m->sources[name] = src;
}

void yx_conv(YPlan* pl, const std::string& name, int src, int s_off, int s_c, int dst, int d_off, int d_c, int h, int w,
             int ks, int stride = 1, int res = -1, int r_off = 0, int act = 1) {
  YStep s; s.kind = YS_CONV; s.w = name; s.src = src; s.s_off = s_off; s.s_c = s_c; s.dst = dst; s.d_off = d_off; s.d_c = d_c;
  s.h = h; s.wd = w; s.ks = ks; s.stride = stride; s.res = res; s.r_off = r_off; s.act = act;
  pl->steps.push_back(s);
}

void yx_base(YoloxModel* m, const std::string& p, int cin, int cout, int k) { yx_conv_decl(m, p, cin, cout, k, {p}); }

// CSPLayer: conv1 / conv2 into the two halves of one concat buffer, bottlenecks in place over the first half (the shortcut
// add after the activation reads and writes each element in the same thread), conv3 from the whole buffer
void yx_csp(YoloxModel* m, YPlan* pl, const std::string& p, int cin, int cout, int n, bool shortcut, int src, int s_off, int dst, int d_off,
            int h, int w) {
  const int hd = cout / 2;
  yx_base(m, p + ".conv1", cin, hd, 1);
  yx_base(m, p + ".conv2", cin, hd, 1);
  yx_base(m, p + ".conv3", 2 * hd, cout, 1);
  const int cat = yx_buf(pl, h, w, 2 * hd);
  yx_conv(pl, p + ".conv1", src, s_off, cin, cat, 0, hd, h, w, 1);
  yx_conv(pl, p + ".conv2", src, s_off, cin, cat, hd, hd, h, w, 1);
  const int tmp = n ? yx_buf(pl, h, w, hd) : -1;
  for (int i = 0; i < n; ++i) {
    const std::string q = p + ".m." + std::to_string(i);
    yx_base(m, q + ".conv1", hd, hd, 1);
    yx_base(m, q + ".conv2", hd, hd, 3);
    yx_conv(pl, q + ".conv1", cat, 0, hd, tmp, 0, hd, h, w, 1);
    yx_conv(pl, q + ".conv2", tmp, 0, hd, cat, 0, hd, h, w, 3, 1, shortcut ? cat : -1, 0);
  }
  yx_conv(pl, p + ".conv3", cat, 0, 2 * hd, dst, d_off, cout, h, w, 1);
}

void yx_build(YoloxModel* m, YPlan* pl) {
  const double depth = m->depth, width = m->width;
  const int b = (int)(width * 64), bd = std::max((int)std::lround(depth * 3), 1), nf = (int)std::lround(3 * depth);
  const int c0 = (int)(256 * width), c1 = (int)(512 * width), c2 = (int)(1024 * width), ch = (int)(256 * width);
  int sh[6], sw[6];
  for (int i = 0; i < 6; ++i) { sh[i] = pl->H >> i; sw[i] = pl->W >> i; }
  const std::string p = "backbone.backbone.";
  YStep f; f.kind = YS_FOCUS;
  f.dst = yx_buf(pl, sh[1], sw[1], 16);
  pl->steps.push_back(f);
  yx_conv_decl(m, p + "stem.conv", 16, b, 3, {p + "stem.conv"});   // 12 Focus channels, padded to 16 with zero weights
  const int x = yx_buf(pl, sh[1], sw[1], b);
  yx_conv(pl, p + "stem.conv", f.dst, 0, 16, x, 0, b, sh[1], sw[1], 3);
  int t = yx_buf(pl, sh[2], sw[2], 2 * b);
  yx_base(m, p + "dark2.0", b, 2 * b, 3);
  yx_conv(pl, p + "dark2.0", x, 0, b, t, 0, 2 * b, sh[1], sw[1], 3, 2);
  const int d2 = yx_buf(pl, sh[2], sw[2], 2 * b);
  yx_csp(m, pl, p + "dark2.1", 2 * b, 2 * b, bd, true, t, 0, d2, 0, sh[2], sw[2]);
  const int cat_p3 = yx_buf(pl, sh[3], sw[3], 2 * c0), cat_p4 = yx_buf(pl, sh[4], sw[4], 2 * c1);
  t = yx_buf(pl, sh[3], sw[3], 4 * b);
  yx_base(m, p + "dark3.0", 2 * b, 4 * b, 3);
  yx_conv(pl, p + "dark3.0", d2, 0, 2 * b, t, 0, 4 * b, sh[2], sw[2], 3, 2);
  yx_csp(m, pl, p + "dark3.1", 4 * b, 4 * b, 3 * bd, true, t, 0, cat_p3, c0, sh[3], sw[3]);     // dark3 -> cat_p3[c0:]
  t = yx_buf(pl, sh[4], sw[4], 8 * b);
  yx_base(m, p + "dark4.0", 4 * b, 8 * b, 3);
  yx_conv(pl, p + "dark4.0", cat_p3, c0, c0, t, 0, 8 * b, sh[3], sw[3], 3, 2);
  yx_csp(m, pl, p + "dark4.1", 8 * b, 8 * b, 3 * bd, true, t, 0, cat_p4, c1, sh[4], sw[4]);     // dark4 -> cat_p4[c1:]
  t = yx_buf(pl, sh[5], sw[5], 16 * b);
  yx_base(m, p + "dark5.0", 8 * b, 16 * b, 3);
  yx_conv(pl, p + "dark5.0", cat_p4, c1, c1, t, 0, 16 * b, sh[4], sw[4], 3, 2);
  const int hs = 8 * b, spp = yx_buf(pl, sh[5], sw[5], 4 * hs);
  yx_base(m, p + "dark5.1.conv1", 16 * b, hs, 1);
  yx_conv(pl, p + "dark5.1.conv1", t, 0, 16 * b, spp, 0, hs, sh[5], sw[5], 1);
  YStep sp; sp.kind = YS_SPP; sp.dst = spp; sp.d_c = hs; sp.h = sh[5]; sp.wd = sw[5];
  pl->steps.push_back(sp);
  const int t2 = yx_buf(pl, sh[5], sw[5], 16 * b);
  yx_base(m, p + "dark5.1.conv2", 4 * hs, 16 * b, 1);
  yx_conv(pl, p + "dark5.1.conv2", spp, 0, 4 * hs, t2, 0, 16 * b, sh[5], sw[5], 1);
  const int d5 = yx_buf(pl, sh[5], sw[5], 16 * b);
  yx_csp(m, pl, p + "dark5.2", 16 * b, 16 * b, bd, false, t2, 0, d5, 0, sh[5], sw[5]);
  // PAFPN (yolo_pafpn.py:82-115)
  const std::string q = "backbone.";
  const int cat_n4 = yx_buf(pl, sh[5], sw[5], 2 * c1), cat_n3 = yx_buf(pl, sh[4], sw[4], 2 * c0);
  yx_base(m, q + "lateral_conv0", c2, c1, 1);
  yx_conv(pl, q + "lateral_conv0", d5, 0, c2, cat_n4, c1, c1, sh[5], sw[5], 1);              // fpn_out0 -> cat_n4[c1:]
  YStep u; u.kind = YS_UP; u.src = cat_n4; u.s_off = c1; u.d_c = c1; u.dst = cat_p4; u.d_off = 0; u.h = sh[5]; u.wd = sw[5];
  pl->steps.push_back(u);
  const int f_out0 = yx_buf(pl, sh[4], sw[4], c1);
  yx_csp(m, pl, q + "C3_p4", 2 * c1, c1, nf, false, cat_p4, 0, f_out0, 0, sh[4], sw[4]);
  yx_base(m, q + "reduce_conv1", c1, c0, 1);
  yx_conv(pl, q + "reduce_conv1", f_out0, 0, c1, cat_n3, c0, c0, sh[4], sw[4], 1);           // fpn_out1 -> cat_n3[c0:]
  u.src = cat_n3; u.s_off = c0; u.d_c = c0; u.dst = cat_p3; u.h = sh[4]; u.wd = sw[4];
  pl->steps.push_back(u);
  const int pan2 = yx_buf(pl, sh[3], sw[3], c0);
  yx_csp(m, pl, q + "C3_p3", 2 * c0, c0, nf, false, cat_p3, 0, pan2, 0, sh[3], sw[3]);
  yx_base(m, q + "bu_conv2", c0, c0, 3);
  yx_conv(pl, q + "bu_conv2", pan2, 0, c0, cat_n3, 0, c0, sh[3], sw[3], 3, 2);
  const int pan1 = yx_buf(pl, sh[4], sw[4], c1);
  yx_csp(m, pl, q + "C3_n3", 2 * c0, c1, nf, false, cat_n3, 0, pan1, 0, sh[4], sw[4]);
  yx_base(m, q + "bu_conv1", c1, c1, 3);
  yx_conv(pl, q + "bu_conv1", pan1, 0, c1, cat_n4, 0, c1, sh[4], sw[4], 3, 2);
  const int pan0 = yx_buf(pl, sh[5], sw[5], c2);
  yx_csp(m, pl, q + "C3_n4", 2 * c1, c2, nf, false, cat_n4, 0, pan0, 0, sh[5], sw[5]);
  // head (yolo_head.py:191-254): cls_convs[k][0] and reg_convs[k][0] as one conv with doubled N; reg + obj as one conv
  const int feats[3] = {pan2, pan1, pan0}, fch[3] = {c0, c1, c2}, strides[3] = {8, 16, 32};
  int a_off = 0;
  for (int k = 0; k < 3; ++k) {
    const int lv = k + 3, h = sh[lv], w = sw[lv];
    const std::string hk = "head.", ks = std::to_string(k);
    const int stem = yx_buf(pl, h, w, ch), both = yx_buf(pl, h, w, 2 * ch), cf = yx_buf(pl, h, w, ch), rf = yx_buf(pl, h, w, ch);
    const int raw = yx_buf(pl, h, w, 5 + m->nc);
    yx_base(m, hk + "stems." + ks, fch[k], ch, 1);
    yx_conv(pl, hk + "stems." + ks, feats[k], 0, fch[k], stem, 0, ch, h, w, 1);
    yx_conv_decl(m, hk + "conv0." + ks, ch, 2 * ch, 3, {hk + "cls_convs." + ks + ".0", hk + "reg_convs." + ks + ".0"});
    yx_conv(pl, hk + "conv0." + ks, stem, 0, ch, both, 0, 2 * ch, h, w, 3);
    yx_base(m, hk + "cls_convs." + ks + ".1", ch, ch, 3);
    yx_base(m, hk + "reg_convs." + ks + ".1", ch, ch, 3);
    yx_conv(pl, hk + "cls_convs." + ks + ".1", both, 0, ch, cf, 0, ch, h, w, 3);
    yx_conv(pl, hk + "reg_convs." + ks + ".1", both, ch, ch, rf, 0, ch, h, w, 3);
    yx_conv_decl(m, hk + "regobj." + ks, ch, 5, 1, {hk + "reg_preds." + ks, hk + "obj_preds." + ks});
    yx_conv_decl(m, hk + "cls." + ks, ch, m->nc, 1, {hk + "cls_preds." + ks});
    yx_conv(pl, hk + "regobj." + ks, rf, 0, ch, raw, 0, 5, h, w, 1, 1, -1, 0, 0);
    yx_conv(pl, hk + "cls." + ks, cf, 0, ch, raw, 5, m->nc, h, w, 1, 1, -1, 0, 0);
    YStep hd; hd.kind = YS_HEAD; hd.src = raw; hd.h = h; hd.wd = w; hd.extra = strides[k]; hd.d_off = a_off;
    pl->steps.push_back(hd);
    a_off += h * w;
  }
  pl->A = a_off;
  pl->offs.resize(pl->bufs.size());
}

// folded float64 weights [cout][cin][k][k] and bias of one source: a BaseConv prefix (conv + bn or fused conv + bias) or a
// prediction conv (weight + bias).  Returns false when a tensor is missing or has the wrong size.
bool yx_source(YoloxModel* m, const std::string& p, int cin, int cout, int k, std::vector<double>& w, std::vector<double>& b) {
  auto get = [&](const std::string& key, size_t n) -> const std::vector<double>* {
    auto it = m->host.find(key);
    return (it != m->host.end() && it->second.size() == n) ? &it->second : nullptr;
  };
  const size_t nw = (size_t)cout * cin * k * k;
  const std::vector<double>* cw = get(p + ".conv.weight", nw);
  if (cw) {
    const std::vector<double>* cb = get(p + ".conv.bias", cout);
    const std::vector<double>* g = get(p + ".bn.weight", cout);
    w = *cw;
    b.assign(cout, 0.0);
    if (g) {   // fuse_conv_and_bn (det/yolox/utils/model_utils.py:33-58), eps 1e-3 (YOLOX.init_yolo)
      const std::vector<double>* be = get(p + ".bn.bias", cout);
      const std::vector<double>* mu = get(p + ".bn.running_mean", cout);
      const std::vector<double>* var = get(p + ".bn.running_var", cout);
      if (!be || !mu || !var) return false;
      for (int o = 0; o < cout; ++o) {
        const double s = (*g)[o] / std::sqrt(1e-3 + (*var)[o]);
        for (size_t i = 0; i < nw / cout; ++i) w[o * (nw / cout) + i] *= s;
        b[o] = s * (cb ? (*cb)[o] : 0.0) + ((*be)[o] - (*g)[o] * (*mu)[o] / std::sqrt((*var)[o] + 1e-3));
      }
      return true;
    }
    if (!cb) return false;
    b = *cb;
    return true;
  }
  const std::vector<double>* pw = get(p + ".weight", nw);
  const std::vector<double>* pb = get(p + ".bias", cout);
  if (!pw || !pb) return false;
  w = *pw;
  b = *pb;
  return true;
}

int yx_pack(YoloxModel* m, const std::string& name, YConv& c, bool& ok) {
  ok = false;
  const std::vector<std::string>& src = m->sources[name];
  const bool regobj = name.find("regobj") != std::string::npos;
  const bool stem = name.size() >= 9 && name.compare(name.size() - 9, 9, "stem.conv") == 0;
  const int src_cin = stem ? 12 : c.cin;   // the Focus output has 12 channels, stored as 16
  std::vector<double> W, Bv;
  for (size_t i = 0; i < src.size(); ++i) {
    const int co = regobj ? (i == 0 ? 4 : 1) : c.cout / (int)src.size();   // reg 4 | obj 1; or [cls | reg] halves
    std::vector<double> w, b;
    if (!yx_source(m, src[i], src_cin, co, c.k, w, b)) return GDRN_OK;
    W.insert(W.end(), w.begin(), w.end());
    Bv.insert(Bv.end(), b.begin(), b.end());
  }
  // [cout][cin'][k][k] -> [cout][(ky, kx, ci)] with cin' padded to c.cin; hi = bf16(w), lo = bf16(w - hi)
  const int K = c.k * c.k * c.cin;
  std::vector<__nv_bfloat16> hi((size_t)c.cout * K), lo((size_t)c.cout * K);
  for (int o = 0; o < c.cout; ++o)
    for (int ky = 0; ky < c.k; ++ky)
      for (int kx = 0; kx < c.k; ++kx)
        for (int ci = 0; ci < c.cin; ++ci) {
          const double v = ci < src_cin ? W[(((size_t)o * src_cin + ci) * c.k + ky) * c.k + kx] : 0.0;
          const __nv_bfloat16 h = __float2bfloat16_rn((float)v);
          const size_t at = (size_t)o * K + (ky * c.k + kx) * c.cin + ci;
          hi[at] = h;
          lo[at] = __float2bfloat16_rn((float)(v - (double)__bfloat162float(h)));
        }
  std::vector<float> bf(Bv.begin(), Bv.end());
  if (!c.hi) {
    GDRN_CHECK_CUDA(cudaMalloc(&c.hi, hi.size() * 2));
    if (m->split) GDRN_CHECK_CUDA(cudaMalloc(&c.lo, lo.size() * 2));
    GDRN_CHECK_CUDA(cudaMalloc(&c.bias, bf.size() * 4));
  }
  GDRN_CHECK_CUDA(cudaMemcpy(c.hi, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
  if (m->split) GDRN_CHECK_CUDA(cudaMemcpy(c.lo, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
  GDRN_CHECK_CUDA(cudaMemcpy(c.bias, bf.data(), bf.size() * 4, cudaMemcpyHostToDevice));
  ok = true;
  c.packed = true;
  return GDRN_OK;
}

int yx_launch_conv(const YoloxModel* m, const YPlan& pl, const YStep& s, const YConv& c, float* const* bp, int B, cudaStream_t st) {
  ConvArgs p;
  p.x = bp[s.src]; p.ldx = pl.bufs[s.src].ld; p.cx_off = s.s_off; p.Cin = s.s_c; p.H = s.h; p.W = s.wd;
  p.w_hi = c.hi; p.w_lo = m->split ? c.lo : nullptr;
  p.K = c.k * c.k * c.cin;
  p.bias = c.bias; p.Cout = c.cout;
  p.ks = c.k; p.stride = s.stride; p.pad = (c.k - 1) / 2;
  p.OH = (s.h + 2 * p.pad - c.k) / s.stride + 1;
  p.OW = (s.wd + 2 * p.pad - c.k) / s.stride + 1;
  p.M = (long long)B * p.OH * p.OW;
  p.out = bp[s.dst]; p.ldo = pl.bufs[s.dst].ld; p.co_off = s.d_off;
  p.resid = s.res >= 0 ? bp[s.res] : nullptr; p.ldr = s.res >= 0 ? pl.bufs[s.res].ld : 0; p.cr_off = s.r_off;
  p.act = s.act;
  const dim3 grid((unsigned)((p.M + CV_BM - 1) / CV_BM), (unsigned)((c.cout + CV_BN - 1) / CV_BN));
  if (m->split) GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_conv_kernel<true>, grid, dim3(CV_THREADS), 0, st, p));
  else GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_conv_kernel<false>, grid, dim3(CV_THREADS), 0, st, p));
  return GDRN_OK;
}

size_t yx_layout(YPlan& pl, int nb) {
  size_t off = 0;
  for (size_t i = 0; i < pl.bufs.size(); ++i) {
    pl.offs[i] = off;
    off += yx_align((size_t)pl.bufs[i].pix * nb * pl.bufs[i].ld * 4);
  }
  return off;
}

// workspace of a forward of B images over the given plans: the largest plan at the first chunk's size
size_t yx_workspace(YoloxModel* m, const std::vector<int>& plans, int B) {
  size_t need = 0;
  for (int k : plans) need = std::max(need, yx_layout(m->plans[k], std::min(B, m->max_batch)));
  return need + 256;
}

bool yx_ready(const YoloxModel* m) {
  for (auto& kv : m->convs)
    if (!kv.second.packed) return false;
  return true;
}

// the buffer pointers of a plan laid out for nb images from the 256-aligned workspace base
int yx_buffers(YPlan& pl, int nb, uint8_t* base, float** bp) {
  GDRN_REQUIRE(pl.bufs.size() <= 512, "yolox_model_forward: too many buffers");
  yx_layout(pl, nb);
  for (size_t i = 0; i < pl.bufs.size(); ++i) bp[i] = reinterpret_cast<float*>(base + pl.offs[i]);
  return GDRN_OK;
}

// one step of a plan over nb images of the original [nb,3,H,W] input x; a head step writes det rows
// [a_base + s.d_off, a_base + s.d_off + h*w) of [nb, A_row, 5 + nc].  One launch.
int yx_run_step(YoloxModel* m, const YPlan& pl, const YStep& s, float* const* bp, const float* x, int nb, float* det, int A_row,
                int a_base, cudaStream_t st) {
  if (s.kind == YS_CONV) return yx_launch_conv(m, pl, s, m->convs.at(s.w), bp, nb, st);
  if (s.kind == YS_FOCUS) {
    const long long n = (long long)nb * (pl.H / 2) * (pl.W / 2);
    if (pl.resample)
      GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_focus_resample_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, st, x, nb, m->H, m->W,
                                      pl.H, pl.W, pl.sh, pl.sw, (float)m->H / (float)pl.sh, (float)m->W / (float)pl.sw, bp[s.dst]));
    else
      GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_focus_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, st, x, nb, pl.H, pl.W, bp[s.dst]));
  } else if (s.kind == YS_SPP) {
    const long long n = (long long)nb * s.h * s.wd * s.d_c;
    GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_spp_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, st, bp[s.dst], nb, s.h, s.wd,
                                    pl.bufs[s.dst].ld, s.d_c));
  } else if (s.kind == YS_UP) {
    const long long n = (long long)nb * 4 * s.h * s.wd * s.d_c;
    GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_upsample2x_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, st,
                                    (const float*)bp[s.src], pl.bufs[s.src].ld, s.s_off, bp[s.dst], pl.bufs[s.dst].ld, s.d_off,
                                    nb, s.h, s.wd, s.d_c));
  } else {
    const long long n = (long long)nb * s.h * s.wd * (5 + m->nc);
    GDRN_CHECK_CUDA(gdrn_launch_dep(yolox_head_out_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, st, (const float*)bp[s.src],
                                    nb, s.h, s.wd, m->nc, s.extra, A_row, a_base + s.d_off, pl.inv_scale, det));
  }
  return GDRN_OK;
}

// one plan over nb images of the original [nb,3,H,W] input x: det rows [a_base, a_base + pl.A) of [nb, A_row, 5 + nc]
int yx_run_plan(YoloxModel* m, YPlan& pl, const float* x, int nb, float* det, int A_row, int a_base, uint8_t* base, cudaStream_t st,
                int& launches) {
  float* bp[512];
  int rc = yx_buffers(pl, nb, base, bp);
  if (rc != GDRN_OK) return rc;
  for (const YStep& s : pl.steps) {
    rc = yx_run_step(m, pl, s, bp, x, nb, det, A_row, a_base, st);
    if (rc != GDRN_OK) return rc;
    ++launches;
  }
  return GDRN_OK;
}

// anchor base of a plan in the rows its forward writes: 0 for plan 0 (yolox_model_forward), the anchors of the scales
// before it for a test-time-augmentation plan (yolox_model_forward_tta); -1 if the plan is not in the scale set
int yx_anchor_base(const YoloxModel* m, int plan) {
  if (plan == 0) return 0;
  int a = 0;
  for (int k : m->tta_plan) {
    if (k == plan) return a;
    a += m->plans[k].A;
  }
  return -1;
}

// the plan of one scale: model_utils.scale_img sizes in double arithmetic from the create-time H x W
int yx_scale_sizes(int H, int W, double s, int* ph, int* pw, int* sh, int* sw) {
  *sh = (int)(H * s);
  *sw = (int)(W * s);
  *ph = (int)(std::ceil(H * s / 32) * 32);
  *pw = (int)(std::ceil(W * s / 32) * 32);
  return *sh >= 1 && *sw >= 1;
}

}  // namespace

extern "C" int yolox_model_create(YoloxModel** out, double depth, double width, int num_classes, int max_batch, int H, int W,
                                  int precision) {
  GDRN_REQUIRE(out, "yolox_model_create: null handle");
  *out = nullptr;
  GDRN_REQUIRE(depth > 0 && width > 0 && num_classes > 0 && max_batch > 0, "yolox_model_create: bad model size");
  GDRN_REQUIRE(H >= 32 && W >= 32 && H % 32 == 0 && W % 32 == 0, "yolox_model_create: H and W must be positive multiples of 32");
  GDRN_REQUIRE(precision == 0 || precision == 1, "yolox_model_create: precision is 1 (bf16x3) or 0 (bf16)");
  const int b = (int)(width * 64), ch = (int)(256 * width);
  GDRN_REQUIRE(b % 8 == 0 && ch % 8 == 0 && (int)(256 * width) == 4 * b && (int)(512 * width) == 8 * b &&
                   (int)(1024 * width) == 16 * b,
               "yolox_model_create: the width must give channel counts that are multiples of 8 (every standard YOLOX width does)");
  YoloxModel* m = new YoloxModel();
  m->nc = num_classes; m->max_batch = max_batch; m->H = H; m->W = W; m->split = precision;
  m->depth = depth; m->width = width;
  m->plans.resize(1);
  YPlan& p0 = m->plans[0];
  p0.H = p0.sh = H; p0.W = p0.sw = W;
  yx_build(m, &p0);
  *out = m;
  return GDRN_OK;
}

extern "C" void yolox_model_destroy(YoloxModel* m) {
  if (!m) return;
  for (auto& kv : m->convs) { cudaFree(kv.second.hi); cudaFree(kv.second.lo); cudaFree(kv.second.bias); }
  delete m;
}

extern "C" int yolox_model_load_tensor(YoloxModel* m, const char* key, const float* data, int64_t numel, void* stream) {
  GDRN_REQUIRE(m && key && (data || numel == 0) && numel >= 0, "yolox_model_load_tensor: bad arguments");
  std::vector<float> f((size_t)numel);
  if (numel) {
    GDRN_CHECK_CUDA(cudaMemcpyAsync(f.data(), data, (size_t)numel * 4, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    GDRN_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  }
  m->host[key].assign(f.begin(), f.end());
  for (auto& kv : m->convs) kv.second.packed = false;   // re-pack at the next yolox_model_missing
  return GDRN_OK;
}

// packs every conv whose tensors are all present; returns the number still missing (or < 0 on a CUDA error)
extern "C" int yolox_model_missing(YoloxModel* m) {
  if (!m) return -1;
  int missing = 0;
  for (auto& kv : m->convs) {
    if (kv.second.packed) continue;
    bool ok = false;
    if (yx_pack(m, kv.first, kv.second, ok) != GDRN_OK) return -1;
    if (!ok) ++missing;
  }
  return missing;
}

extern "C" int yolox_model_num_anchors(const YoloxModel* m) { return m ? m->plans[0].A : 0; }

extern "C" size_t yolox_model_workspace_bytes(YoloxModel* m, int B) {
  if (!m || B <= 0) return 0;
  return yx_workspace(m, {0}, B);
}

extern "C" int yolox_model_forward(YoloxModel* m, const float* img, int B, float* det_preds, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  GDRN_REQUIRE(m && img && det_preds && workspace && B > 0, "yolox_model_forward: bad arguments");
  GDRN_REQUIRE(yx_ready(m), "yolox_model_forward: weights missing (load every tensor, then yolox_model_missing)");
  GDRN_REQUIRE(workspace_bytes >= yx_workspace(m, {0}, B), "yolox_model_forward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  YPlan& pl = m->plans[0];
  const int C = 5 + m->nc;
  int launches = 0;
  for (int i0 = 0; i0 < B; i0 += m->max_batch) {
    const int nb = std::min(m->max_batch, B - i0);
    const int rc = yx_run_plan(m, pl, img + (size_t)i0 * 3 * m->H * m->W, nb, det_preds + (size_t)i0 * pl.A * C, pl.A, 0, base, st,
                               launches);
    if (rc != GDRN_OK) return rc;
  }
  gdrn_count_launch(launches);
  return GDRN_OK;
}

// Multi-scale test-time augmentation (YOLOX.forward(augment=True)).  Host only: plans are layer lists over the shared
// packed weights, so nothing is allocated on the device and no weight is re-packed.  A scale of exactly 1.0 reuses plan 0.
extern "C" int yolox_model_set_scales(YoloxModel* m, const double* scales, int n_scales) {
  GDRN_REQUIRE(m && scales && n_scales > 0, "yolox_model_set_scales: bad arguments");
  for (int i = 0; i < n_scales; ++i) {
    int ph, pw, sh, sw;
    GDRN_REQUIRE(std::isfinite(scales[i]) && scales[i] > 0 && yx_scale_sizes(m->H, m->W, scales[i], &ph, &pw, &sh, &sw),
                 "yolox_model_set_scales: a scale gives an empty resampled image (int(H * s) or int(W * s) is 0)");
  }
  m->plans.resize(1);
  m->tta_plan.clear();
  m->A_tta = 0;
  for (int i = 0; i < n_scales; ++i) {
    const double s = scales[i];
    if (s == 1.0) {
      m->tta_plan.push_back(0);
    } else {
      YPlan pl;
      yx_scale_sizes(m->H, m->W, s, &pl.H, &pl.W, &pl.sh, &pl.sw);
      pl.resample = true;
      pl.inv_scale = 1.0f / (float)s;
      yx_build(m, &pl);
      m->plans.push_back(std::move(pl));
      m->tta_plan.push_back((int)m->plans.size() - 1);
    }
    m->A_tta += m->plans[m->tta_plan.back()].A;
  }
  return GDRN_OK;
}

extern "C" int yolox_model_num_anchors_tta(const YoloxModel* m) { return m ? m->A_tta : 0; }

extern "C" size_t yolox_model_workspace_bytes_tta(YoloxModel* m, int B) {
  if (!m || B <= 0 || m->tta_plan.empty()) return 0;
  return yx_workspace(m, m->tta_plan, B);
}

extern "C" int yolox_model_forward_tta(YoloxModel* m, const float* img, int B, float* det_preds, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  GDRN_REQUIRE(m && img && det_preds && workspace && B > 0, "yolox_model_forward_tta: bad arguments");
  GDRN_REQUIRE(!m->tta_plan.empty(), "yolox_model_forward_tta: no scales (call yolox_model_set_scales first)");
  GDRN_REQUIRE(yx_ready(m), "yolox_model_forward_tta: weights missing (load every tensor, then yolox_model_missing)");
  GDRN_REQUIRE(workspace_bytes >= yx_workspace(m, m->tta_plan, B), "yolox_model_forward_tta: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  const int C = 5 + m->nc;
  int launches = 0;
  for (int i0 = 0; i0 < B; i0 += m->max_batch) {
    const int nb = std::min(m->max_batch, B - i0);
    const float* x = img + (size_t)i0 * 3 * m->H * m->W;
    float* det = det_preds + (size_t)i0 * m->A_tta * C;
    int a_base = 0;
    for (int k : m->tta_plan) {   // the scales in order, one after the other in the same workspace
      const int rc = yx_run_plan(m, m->plans[k], x, nb, det, m->A_tta, a_base, base, st, launches);
      if (rc != GDRN_OK) return rc;
      a_base += m->plans[k].A;
    }
  }
  gdrn_count_launch(launches);
  return GDRN_OK;
}

// ---- test / measurement entries: walk a plan's step table and run one step of it (include/gdrn_b200.h) ----
extern "C" int yolox_model_plan_info(YoloxModel* m, int plan, int* info) {
  GDRN_REQUIRE(m && info, "yolox_model_plan_info: bad arguments");
  GDRN_REQUIRE(plan >= 0 && plan < (int)m->plans.size(), "yolox_model_plan_info: no such plan");
  const YPlan& pl = m->plans[plan];
  const int v[9] = {(int)pl.steps.size(), (int)pl.bufs.size(), pl.H, pl.W, pl.sh, pl.sw, pl.A,
                    plan == 0 ? pl.A : m->A_tta, yx_anchor_base(m, plan)};
  for (int i = 0; i < 9; ++i) info[i] = v[i];
  return GDRN_OK;
}

extern "C" int yolox_model_step_info(YoloxModel* m, int plan, int step, int* info, char* name, int name_len) {
  GDRN_REQUIRE(m && info && name && name_len > 0, "yolox_model_step_info: bad arguments");
  GDRN_REQUIRE(plan >= 0 && plan < (int)m->plans.size(), "yolox_model_step_info: no such plan");
  const YPlan& pl = m->plans[plan];
  GDRN_REQUIRE(step >= 0 && step < (int)pl.steps.size(), "yolox_model_step_info: no such step");
  const YStep& s = pl.steps[step];
  GDRN_REQUIRE((int)s.w.size() < name_len, "yolox_model_step_info: name buffer too small");
  const int C = 5 + m->nc;
  // kind, src, s_off, s_c, dst, d_off, d_c, res, r_off, in h, in w, out h, out w, ks, stride, act, level stride, anchor offset
  int v[18] = {s.kind, s.src, s.s_off, s.s_c, s.dst, s.d_off, s.d_c, s.res, s.r_off, s.h, s.wd, s.h, s.wd, 0, 0, 0, 0, 0};
  if (s.kind == YS_CONV) {
    const int k = m->convs.at(s.w).k, pad = (k - 1) / 2;
    v[11] = (s.h + 2 * pad - k) / s.stride + 1;
    v[12] = (s.wd + 2 * pad - k) / s.stride + 1;
    v[13] = k; v[14] = s.stride; v[15] = s.act;
  } else if (s.kind == YS_FOCUS) {   // reads the [B,3,H,W] input (the create-time size: a scaled plan resamples it)
    v[1] = -1; v[2] = 0; v[3] = 3; v[6] = 16; v[9] = m->H; v[10] = m->W; v[11] = pl.H / 2; v[12] = pl.W / 2;
  } else if (s.kind == YS_SPP) {     // pools slice [0, C) of its buffer into slices C, 2C, 3C
    v[1] = s.dst; v[2] = 0; v[3] = s.d_c; v[5] = s.d_c; v[6] = 3 * s.d_c; v[13] = 13; v[14] = 1;
  } else if (s.kind == YS_UP) {
    v[3] = s.d_c; v[11] = 2 * s.h; v[12] = 2 * s.wd;
  } else {                           // reads the level's raw buffer, writes det rows
    v[2] = 0; v[3] = C; v[4] = -1; v[5] = 0; v[6] = C; v[16] = s.extra; v[17] = s.d_off;
  }
  for (int i = 0; i < 18; ++i) info[i] = v[i];
  std::memcpy(name, s.w.c_str(), s.w.size() + 1);
  return GDRN_OK;
}

extern "C" int yolox_model_buffer_info(YoloxModel* m, int plan, int buf, int batch, int64_t* info) {
  GDRN_REQUIRE(m && info, "yolox_model_buffer_info: bad arguments");
  GDRN_REQUIRE(plan >= 0 && plan < (int)m->plans.size(), "yolox_model_buffer_info: no such plan");
  YPlan& pl = m->plans[plan];
  GDRN_REQUIRE(buf >= 0 && buf < (int)pl.bufs.size(), "yolox_model_buffer_info: no such buffer");
  GDRN_REQUIRE(batch > 0 && batch <= m->max_batch, "yolox_model_buffer_info: batch must be 1..max_batch");
  const size_t need = yx_layout(pl, batch) + 256;
  info[0] = (int64_t)pl.offs[buf];
  info[1] = pl.bufs[buf].pix;
  info[2] = pl.bufs[buf].ld;
  info[3] = (int64_t)need;
  return GDRN_OK;
}

extern "C" int yolox_model_run_step(YoloxModel* m, int plan, int step, const float* img, int batch, float* det_preds, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(m && img && det_preds && workspace, "yolox_model_run_step: bad arguments");
  GDRN_REQUIRE(plan >= 0 && plan < (int)m->plans.size(), "yolox_model_run_step: no such plan");
  YPlan& pl = m->plans[plan];
  GDRN_REQUIRE(step >= 0 && step < (int)pl.steps.size(), "yolox_model_run_step: no such step");
  GDRN_REQUIRE(batch > 0 && batch <= m->max_batch, "yolox_model_run_step: batch must be 1..max_batch");
  GDRN_REQUIRE(yx_ready(m), "yolox_model_run_step: weights missing (load every tensor, then yolox_model_missing)");
  const int a_base = yx_anchor_base(m, plan);
  GDRN_REQUIRE(a_base >= 0, "yolox_model_run_step: the plan is not in the scale set");
  GDRN_REQUIRE(workspace_bytes >= yx_layout(pl, batch) + 256, "yolox_model_run_step: workspace too small");
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  float* bp[512];
  int rc = yx_buffers(pl, batch, base, bp);
  if (rc != GDRN_OK) return rc;
  rc = yx_run_step(m, pl, pl.steps[step], bp, img, batch, det_preds, plan == 0 ? pl.A : m->A_tta, a_base, (cudaStream_t)stream);
  if (rc != GDRN_OK) return rc;
  gdrn_count_launch(1);
  return GDRN_OK;
}

// workspace layout, byte offsets from the 256-byte-aligned base: score [B,A] f32, cls [B,A] i32, sel [B,nc] i32
static void ksi_layout(int B, int A, size_t off[3]) {
  off[0] = 0;
  off[1] = ((size_t)B * A * 4 + 255) & ~(size_t)255;
  off[2] = off[1] + (((size_t)B * A * 4 + 255) & ~(size_t)255);
}

extern "C" size_t yolox_postprocess_single_workspace_bytes(int B, int A, int num_classes) {
  if (B <= 0 || A <= 0 || num_classes <= 0) return 0;
  return (size_t)B * A * 8 + (size_t)B * num_classes * 4 + 4 * 256;
}

extern "C" int yolox_postprocess_single_layout(int B, int A, int num_classes, size_t* offsets) {
  GDRN_REQUIRE(offsets && B > 0 && A > 0 && num_classes > 0, "yolox_postprocess_single_layout: bad arguments");
  ksi_layout(B, A, offsets);
  return GDRN_OK;
}

extern "C" int yolox_postprocess_single(const float* preds, int B, int A, int num_classes, float conf_thre, double nms_thre,
                                        float* dets, int* n_det, void* workspace, size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(preds && dets && n_det && workspace, "yolox_postprocess_single: null argument");
  GDRN_REQUIRE(B > 0 && A > 0 && num_classes > 0 && num_classes <= KSI_MAX_CLASSES, "yolox_postprocess_single: bad problem size");
  GDRN_REQUIRE(workspace_bytes >= yolox_postprocess_single_workspace_bytes(B, A, num_classes),
               "yolox_postprocess_single: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  size_t off[3];
  ksi_layout(B, A, off);
  float* score = reinterpret_cast<float*>(base + off[0]);
  int* cls = reinterpret_cast<int*>(base + off[1]);
  int* sel = reinterpret_cast<int*>(base + off[2]);
  yolox_ksi_score_kernel<<<blocks_for((long long)B * A, 256), 256, 0, st>>>(preds, B, A, num_classes, score, cls);
  yolox_ksi_select_kernel<<<dim3(num_classes, B), 256, 0, st>>>(score, cls, A, num_classes, conf_thre, sel);
  yolox_ksi_nms_kernel<<<B, 1, 0, st>>>(preds, sel, score, A, num_classes, nms_thre, dets, n_det);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(3);
  return GDRN_OK;
}
