// Internal launchers of the CUDA-core kernels around the wgmma GEMMs (dense_ops.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

// generic strided repack (weights): dst[doff + sum i_k*ds_k] = src[soff + sum i_k*ss_k], i_k < dims[k]
struct PackDesc {
  long long dims[4];
  long long ss[4];
  long long ds[4];
  long long soff, doff;
  long long lo_delta;  // > 0 (bf16 dst): also write lo = bf16(v - float(hi)) at dst offset + lo_delta (split-bf16 weights)
};
int launch_pack(const float* src, void* dst, int dst_is_bf16, const PackDesc& d, cudaStream_t st);

// stem: NCHW fp32 image -> bf16 patch rows [B*(H/4)*(W/4), 64] (k = c*16 + ky*4 + kx, 48..63 zero)
int launch_stem_patchify(const float* img, __nv_bfloat16* out, int B, int H, int W, int split, cudaStream_t st);

// ConvNeXt block front half: depthwise 7x7 (pad 3) + bias, LayerNorm over C (eps) -> bf16 [B*H*W, C]
// x: fp32 NHWC; w: [49][C] (tap-major, repacked); all fp32.
// c_real (0 = C): the tensor carries C - c_real trailing zero PAD channels (zero filter taps / bias / LN affine), e.g. the
// 96-channel stage of convnext_tiny/small stored 128 wide; LayerNorm statistics are taken over the c_real channels.
// variant -1 picks the kernel from the shape: the persistent ping-pong kernel when B * (H/8) * (W/16) >= 32 and it takes
// the shape, else the 16x8-pixel x 64-channel cluster kernel (H % 8 == 0, W % 16 == 0, C <= 512), else the 8x8 x 128 one
// (H % 8 == 0, W % 8 == 0, C % 128 == 0).  0 = cluster kernel, 1 = ping-pong kernel.  Other shapes: GDRN_ERR_INVALID.
int launch_dwconv_ln(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                     __nv_bfloat16* out, int B, int H, int W, int C, float eps, int split, int variant, cudaStream_t st,
                     int c_real = 0);
// persistent two-warpgroup ping-pong version (dwconv_pp.cu) for 16x8x64 tiles; returns 1 if the shape is not handled
int launch_dwconv_ln_pp(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                        __nv_bfloat16* out, int B, int H, int W, int C, float eps, int split, cudaStream_t st, int c_real = 0);
// the tensor maps both depthwise kernels load through: x [B,H,W,C] in (cpc x box_w x box_h) halo boxes (out-of-bounds
// zero fill) and w49c [49][C] in (cpc x 49) boxes
int make_dwconv_tmaps(CUtensorMap* tmap_x, CUtensorMap* tmap_w, const float* x, const float* w49c, int B, int H, int W,
                      int C, int cpc, int box_w, int box_h);

// downsample front half: per-pixel LayerNorm over C then 2x2/s2 patchify -> bf16 [B*(H/2)*(W/2), 4*C]
// (k = (ky*2+kx)*C + c)
int launch_ln_patchify2(const float* x, const float* ln_w, const float* ln_b, __nv_bfloat16* out, int B, int H, int W,
                        int C, float eps, int split, cudaStream_t st, int c_real = 0);

int launch_cast_bf16(const float* src, __nv_bfloat16* dst, long long n, cudaStream_t st);

// GroupNorm apply + GELU on NHWC.  raw: bf16 or fp32 [B,h,w,C]; stats: double [B,G,2] (sum, sumsq over h*w*cpg);
// out bf16 [B,h,w,C].
int launch_gn_gelu(const void* raw, int raw_is_f32, const double* stats, float* mean_rstd_scratch /*[B*groups*2]*/,
                   const float* gn_w, const float* gn_b, __nv_bfloat16* out, int B, int h, int w, int C, int groups, float eps,
                   int split, cudaStream_t st);
int launch_gn_gelu_f32(const float* raw, const double* stats, float* mean_rstd_scratch, const float* gn_w,
                       const float* gn_b, float* out, int B, int h, int w, int C, int groups, float eps, cudaStream_t st);
// fp32 CUDA-core fully connected layer (split-bf16 mode FC stack): y[b,n] = act(x[b,:] . W[n,:] + bias[n])
// part: scratch of fc_f32_part_bytes(B, N) bytes (partial sums of the K slices)
int launch_fc_f32(const float* x, const float* W, const float* bias, float* y, float* part, int B, int N, int K, int ldy, int gelu,
                  cudaStream_t st);
size_t fc_f32_part_bytes(int B, int N_max);
// fp32 [rows,C] -> split bf16 [rows,2C]
int launch_cast_split(const float* src, __nv_bfloat16* dst, long long rows, int C, cudaStream_t st);
// bilinear x2 (align_corners=True) on NHWC bf16: [B,h,w,C] -> [B,2h,2w,C]
int launch_upsample2x(const __nv_bfloat16* in, __nv_bfloat16* out, int B, int h, int w, int C, int split, cudaStream_t st);

// rot6d -> R_allo, centroid/z -> t, allocentric -> egocentric. raw: [B, ld] fp32 (rot6d at 0..5, t_ at 6..8)
int launch_pose_lift(const float* raw, int ld, const float* cams, const float* centers, const float* whs,
                     const float* ratios, float* out_rot, float* out_trans, float* out_raw9, int B, cudaStream_t st);

// debug: bf16 -> fp32 copy
int launch_bf16_to_f32(const __nv_bfloat16* src, float* dst, long long n, cudaStream_t st);
// debug: split bf16 [rows, 2C] ([hi C | lo C]) -> fp32 [rows, C] = hi + lo
int launch_split_to_f32(const __nv_bfloat16* src, float* dst, long long rows, int C, cudaStream_t st);
