/* libgdrn_b200.so -- C ABI of the H100-native GDRNPP per-ROI pose-inference hot path.
 *
 * Plain pointers and sizes only (no torch types).  Unless stated otherwise every pointer is a DEVICE
 * pointer, every call is asynchronous on the given CUDA stream (passed as void* = cudaStream_t), never
 * allocates, never synchronises, and returns 0 (GDRN_OK) or a negative error code; the message of the
 * last error is available from gdrn_last_error().  One process per GPU; the caller owns all buffers.
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference tree
 * shanice-l/gdrnpp_bop2022 @ b80383bd).  The reference-side bindings are shown in INTEGRATION.md.
 */
#ifndef GDRN_B200_H_
#define GDRN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GDRN_OK 0
#define GDRN_ERR_INVALID (-1) /* bad argument / unsupported configuration */
#define GDRN_ERR_CUDA (-2)    /* CUDA runtime or driver error */
#define GDRN_ERR_STATE (-3)   /* model not fully loaded, workspace too small, ... */

const char* gdrn_last_error(void);
int gdrn_version(void);
/* number of CUDA kernels this library has launched in the calling process (monotonic) */
long long gdrn_launch_count(void);
/* Which implicit-GEMM kernels this library has launched in the calling process since the last reset: bit i is set once
 * kernel i ran (i numbers the instantiations of the kGemmKernels table in gemm_tc.cu, then the two fused ConvNeXt MLP
 * kernels; gdrnpp_bop2022_b200._lib.GEMM_KERNELS names them).  reset != 0 clears the record after reading it.
 * Host-side bookkeeping only: no launch and no result depends on it. */
uint64_t gdrn_gemm_kernels_launched(int reset);

/* ---------------------------------------------------------------------------------------------
 * Dense path: GDRN_DoubleMask.forward (eval, do_loss=False)
 *   replaces core/gdrn_modeling/models/GDRN_double_mask.py:66-214 and everything it calls:
 *   timm convnext features (core/utils/timm_utils.py:9-35), TopDownDoubleMaskXyzRegionHead.forward
 *   (models/heads/top_down_doublemask_xyz_region_head.py:177-211), ConvPnPNet.forward
 *   (models/heads/conv_pnp_net.py:120-183), rot6d_to_mat_batch (core/utils/rot_reps.py:34-55),
 *   pose_from_predictions_test (models/pose_from_pred_centroid_z.py:56-154) and
 *   allocentric_to_egocentric (core/utils/utils.py:31-88).
 * ------------------------------------------------------------------------------------------- */
typedef struct GdrnModel GdrnModel;

/* arch: "convnext_base" | "convnext_small" | "convnext_tiny"; num_classes: class-aware head size (21), or 1 for the
 * class-agnostic head of the reference's per-object models (XYZ/MASK/REGION_CLASS_AWARE all false: out_layer
 * [70,256,1,1], channels vis 0, full 1, x/y/z 2..4, region 5..69). */
int gdrn_model_create(GdrnModel** out, const char* arch, int num_classes, int max_batch);
/* precision: 0 = bf16 tensor-core operands, fp32 accumulate / residual stream (the throughput mode; what the
 *               reference's AMP test path does, engine_utils.py autocast);
 *            1 = split-bf16 ("bf16x3"): every GEMM operand is the pair (hi, lo) of bf16 values and every GEMM
 *               accumulates A_lo*W_hi + A_hi*W_lo + A_hi*W_hi in fp32; exact-erf GELU; fp32 Patch-PnP FC stack.
 *               Reproduces the reference's fp32 forward to ~1e-5 relative (the BASELINE.json parity bar).
 * gdrn_model_create() uses precision 0 unless the environment variable GDRN_PRECISION says otherwise. */
int gdrn_model_create_ex(GdrnModel** out, const char* arch, int num_classes, int max_batch, int precision);
int gdrn_model_precision(const GdrnModel* m);
void gdrn_model_destroy(GdrnModel* m);

/* Feed one fp32 tensor of a reference checkpoint (state_dict key names, e.g.
 * "backbone.stages_2.blocks.5.mlp.fc1.weight", "geo_head_net.features.0.weight", "pnp_net.fc_r.bias";
 * loader: core/utils/my_checkpoint.py:35-83).  The tensor is re-packed into kernel-native layouts on
 * `stream`; the source buffer may be freed after the stream reaches this point. Unknown keys return
 * GDRN_ERR_INVALID. */
int gdrn_model_load_tensor(GdrnModel* m, const char* key, const float* data, int64_t numel, void* stream);
/* number of tensors still missing (0 = ready) */
int gdrn_model_missing(const GdrnModel* m);

size_t gdrn_model_workspace_bytes(const GdrnModel* m, int batch);

typedef struct GdrnMaps { /* optional class-gathered maps (GDRN_double_mask.py:203-214), fp32 NCHW, or all NULL */
  float* mask;      /* [B,1,64,64] */
  float* full_mask; /* [B,1,64,64] */
  float* coor_x;    /* [B,1,64,64] */
  float* coor_y;    /* [B,1,64,64] */
  float* coor_z;    /* [B,1,64,64] */
  float* region;    /* [B,65,64,64] */
} GdrnMaps;

/* roi_img [B,3,256,256] fp32 NCHW in [0,1]; roi_classes [B] int64; roi_coord_2d [B,2,64,64]; roi_cams [B,3,3];
 * roi_centers [B,2]; roi_whs [B,2]; resize_ratios [B]; roi_extents [B,3]  ->  out_rot [B,3,3] (egocentric,
 * row-major), out_trans [B,3].  out_raw (optional, [B,9]) receives the Patch-PnP head output (rot6d, t_).
 * roi_classes may be NULL only for a model created with num_classes = 1 (class-agnostic head): the head then reads
 * no labels and every ROI uses the one class slab.  A class-aware model rejects NULL with GDRN_ERR_INVALID.  Non-NULL
 * labels are clamped into [0, num_classes) as before. */
int gdrn_model_forward(GdrnModel* m, const float* roi_img, const int64_t* roi_classes, const float* roi_coord_2d,
                       const float* roi_cams, const float* roi_centers, const float* roi_whs,
                       const float* resize_ratios, const float* roi_extents, int batch, float* out_rot,
                       float* out_trans, float* out_raw, const GdrnMaps* maps, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Per-category device timing of the LAST forward (CUDA events on the launch stream): categories
 * 0 = wgmma GEMM kernel, 1 = depthwise-7x7+LayerNorm kernel, 2 = other CUDA-core kernels.
 * get_profile blocks until that forward has finished. */
int gdrn_model_set_profiling(GdrnModel* m, int enable);
int gdrn_model_get_profile(GdrnModel* m, float* ms_out, int* launches_out);

/* debugging / parity hooks: copy an internal activation (after the last forward on the same workspace)
 * as fp32 into dst.  name: "stage3_x" ([B,8,8,C3] NHWC, the fp32 backbone output) | "fc_out" ([B,16], rows 0-5 rot6d,
 * 6-8 t_) | "conv_feat" ([B,8,8,C3], the bf16 backbone output) | "head64" ([B,64,64,256], last head conv after GN+GELU) |
 * "pnp_in" ([B,64,64,128]) | "pnp_feat" ([B,8192]).  Split-bf16 mode reads "stage3_x" and "fc_out" only.
 * C3 as in gdrn_model_run_stage.  Returns element count or <0. */
int64_t gdrn_model_debug_read(GdrnModel* m, const char* name, int batch, float* dst, void* workspace, void* stream);

/* Test / measurement entry: runs ONE backbone, geometry-head or Patch-PnP stage of gdrn_model_forward -- the same host
 * function, plans and kernels the forward launches -- on the model's packed weights, in a gdrn_model_workspace_bytes(m, batch)
 * workspace.  Head / Patch-PnP stages: the fp32 input is first cast to the stage's operand format (bf16, or [hi | lo] split
 * rows in split-bf16 mode); the outputs are decoded to fp32 (hi + lo).  Backbone stages: the residual stream is fp32 in both
 * modes, so input and output are copied unchanged.  All tensors NHWC unless noted.
 *   stage          in                       out
 *   "stem"         [B,3,256,256] NCHW       [B,64,64,cp0]      4x4 s4 conv + LayerNorm2d
 *   "down<s>"      [B,2r,2r,cp[s-1]],       [B,r,r,cp[s]]      LayerNorm2d + 2x2 s2 conv; raw_out: the GEMM operand
 *                  s = 1..3, r = 64>>s                         [B,r,r,4*cp[s-1]] (LayerNorm output, 2x2 patch rows)
 *   "block<s>_<i>" [B,r,r,cp[s]], r = 64>>s [B,r,r,cp[s]]      ConvNeXt block i of stage s (i < depth, e.g. "block2_26");
 *                                                              raw_out: the GEMM operand [B,r,r,cp[s]] (dwconv + LayerNorm)
 *   "deconv"       [B,8,8,C3]               [B,16,16,256]      3x3 s2 transposed conv + GroupNorm + GELU
 *   "head_conv<i>" [B,h,h,256], i = 0..5,   [B,h',h',256]      3x3 conv + GroupNorm + GELU (+ bilinear x2 after i = 1, 3)
 *                  h = 16,16,32,32,64,64
 *   "out_conv"     [B,64,64,256]            [B,64,64,128]      class-gathered 1x1 conv -> Patch-PnP input (69 channels +
 *                                                              zero pad); maps (optional, NCHW) as in gdrn_model_forward
 *   "pnp_conv<i>"  [B,2r,2r,128], r = 32>>i [B,r,r,128]        3x3 s2 conv + GroupNorm + GELU
 *   "pnp_fc"       [B,8,8,128]              [B,16]             fc1 -> fc2 -> fc_r | fc_t (rows 0-5 rot6d, 6-8 t_, rest 0)
 * cp[s] is the stored width of backbone stage s: its channel count rounded up to a multiple of 64 (convnext_tiny / small:
 * 128, 192, 384, 768 for 96, 192, 384, 768 channels); the pad channels are zero.  C3 = cp[3] (1024 for convnext_base).
 * Backbone stages take no gn_stats_out.  For the head conv stages, raw_out (optional) receives the conv
 * output before GroupNorm (at the conv's resolution) and gn_stats_out (optional) the whole table of GroupNorm sums
 * [10][B][32][2] (layer: 0 deconv, 1-6 head convs, 7-9 Patch-PnP convs; per (image, group): sum, sum of squares), cleared
 * before the stage runs.  roi_classes / roi_extents / roi_coord_2d as in gdrn_model_forward, read by "out_conv" only.
 * No allocation, no synchronisation. */
int gdrn_model_run_stage(GdrnModel* m, const char* stage, int batch, const float* in, float* out, float* raw_out,
                         double* gn_stats_out, const int64_t* roi_classes, const float* roi_extents,
                         const float* roi_coord_2d, const GdrnMaps* maps, void* workspace, size_t workspace_bytes,
                         void* stream);

/* Test / measurement entries of the YOLOX engine (yolox_model_*, below): walk the layer plan of a forward and run ONE of
 * its steps -- the same host function and kernel the forward launches for it -- on a caller's workspace.  plan indexes the
 * engine's plans: 0 is the create-time size (yolox_model_forward), 1.. the non-unit scales of the current
 * yolox_model_set_scales set in the order they were added (yolox_model_forward_tta).  Buffers are fp32 NHWC
 * [batch, pix, ld] at an offset from the workspace pointer rounded up to 256 bytes.
 *   yolox_model_plan_info: info[9] = {n_steps, n_buffers, H, W, content h, content w (= H, W for plan 0), A (the plan's
 *     anchors), A_row (det_preds row count the forward writes: A for plan 0, A_tta otherwise), anchor base of the plan}.
 *   yolox_model_step_info: info[18] =
 *      0 kind (0 conv, 1 Focus, 2 SPP, 3 nearest x2 upsample, 4 head output)
 *      1 src buffer (-1: the [B,3,H,W] input), 2 src channel offset, 3 src channel count,
 *      4 dst buffer (-1: det_preds), 5 dst channel offset, 6 dst channel count,
 *      7 residual buffer (-1: none; conv only, added after the activation), 8 residual channel offset,
 *      9 / 10 input map h / w, 11 / 12 output map h / w, 13 kernel size (conv; 13 for SPP), 14 stride (conv, SPP),
 *     15 SiLU flag (conv), 16 level stride (head), 17 anchor offset of the level within the plan (head).
 *     SPP reads slice [0, C) of its buffer and writes slices C, 2C, 3C (dst offset C, count 3C).  The head step reads
 *     the level's raw [pix, 5 + nc] buffer and writes det rows anchor base + anchor offset + [0, h*w).  name (name_len
 *     bytes) receives the packed conv name ("backbone.backbone.dark2.0", "head.conv0.1" = [cls_convs.1.0 | reg_convs.1.0]
 *     along N, "head.regobj.2" = [reg_preds.2 | obj_preds.2], "head.cls.0" = cls_preds.0), "" for other kinds.
 *   yolox_model_buffer_info: info[4] = {byte offset from the aligned base, pixels per image, ld (channels), workspace bytes
 *     the plan needs} for a chunk of batch <= max_batch images, laid out as the forward lays it out.
 *   yolox_model_run_step: step of plan for batch <= max_batch images of img [batch,3,H,W]; a head step writes det_preds
 *     rows of stride A_row at the plan's anchor base.  Rejects a bad plan / step index, a batch above max_batch, a
 *     workspace smaller than the plan needs and missing weights.  No allocation, no synchronisation. */
typedef struct YoloxModel YoloxModel;
int yolox_model_plan_info(YoloxModel* m, int plan, int* info);
int yolox_model_step_info(YoloxModel* m, int plan, int step, int* info, char* name, int name_len);
int yolox_model_buffer_info(YoloxModel* m, int plan, int buf, int batch, int64_t* info);
int yolox_model_run_step(YoloxModel* m, int plan, int step, const float* img, int batch, float* det_preds, void* workspace,
                         size_t workspace_bytes, void* stream);

/* Plain GEMM through the same wgmma kernel, exported for tests and roofline measurement:
 * out[M,N] = epi(A[M,K] @ W[N,K]^T + bias); A, W bf16 row-major (K contiguous, lda/ldw = K).
 * epi: 0 = store (out bf16 or fp32 by out_f32), 1 = GELU -> bf16, 2 = resid + gamma*(.) -> fp32. */
int gdrn_gemm_bf16(const void* A, const void* W, const float* bias, const float* gamma, const float* resid,
                   void* out, int M, int N, int K, int epi, int out_f32, int block_n, void* stream);

/* The same for the split-bf16 ("bf16x3") precision mode, exported for tests and roofline measurement:
 * A [M, 2K] and W [N, 2K] hold [hi K | lo K] rows (hi = bf16(v), lo = bf16(v - hi)); the kernel accumulates
 * A_lo*W_hi + A_hi*W_lo + A_hi*W_hi in fp32.  epi: 0 = store fp32 [M,N]; 1 = exact-erf GELU -> split bf16 [M, 2N];
 * 2 = resid + gamma*(.) -> fp32 [M,N] (in place allowed).  block_n in {64, 128, 256}; N % 64 == 0, K % 64 == 0.
 * epi 1 needs a 16-byte aligned out (GDRN_ERR_INVALID otherwise); epi 0 and 2 need 8-byte aligned out and resid. */
int gdrn_gemm_x3(const void* A, const void* W, const float* bias, const float* gamma, const float* resid, void* out,
                 int M, int N, int K, int epi, int block_n, void* stream);

/* Fused ConvNeXt MLP half-block of the split-bf16 mode (stage 0, C = 128), exported for tests and measurement:
 * x [M,C] fp32 += gamma * (W2 . gelu(W1 . a + b1) + b2) with a [M,2C], W1 [4C,2C], W2 [C,8C] in [hi | lo] bf16 rows; the
 * 4C-wide hidden activation stays on chip.  Replaces two gdrn_gemm_x3 calls (epi 1 then epi 2); same arithmetic.
 * Reference op: timm ConvNeXtBlock.mlp + layer scale + shortcut (models/GDRN_double_mask.py:102 via the backbone). */
int gdrn_mlp_fused_x3(const void* A, const void* W1, const float* b1, const void* W2, const float* b2, const float* gamma,
                      float* x, long long M, int C, void* stream);

/* ConvNeXt block front half exported for tests and roofline measurement: depthwise 7x7 (pad 3) + bias + LayerNorm(C)
 * on an NHWC fp32 tensor x [B,H,W,C] with tap-major weights w49c [49][C] -> bf16 [B*H*W, C] (split = 1: [hi C | lo C]).
 * variant: -1 default, 0 = one-tile-per-CTA cluster kernel, 1 = persistent two-warpgroup ping-pong kernel.
 * Supported shapes: C a multiple of 64 up to 1024, H % 8 == 0, and either W % 16 == 0 with C <= 512 or W % 8 == 0 with
 * C % 128 == 0; variant 1 also needs W % 16 == 0 and C / 64 in {2, 3, 4, 6, 8}.  The default takes the ping-pong kernel
 * when B * (H/8) * (W/16) >= 32 and the shape allows it.  Any other shape or variant returns GDRN_ERR_INVALID before
 * anything is launched. */
int gdrn_dwconv_ln(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b, void* out,
                   int B, int H, int W, int C, float eps, int split, int variant, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Farthest point sampling -- replaces core/csrc/fps/src/farthest_point_sampling.cpp:166-204
 * (cffi surface core/csrc/fps/src/ext.h:1-14, Python wrapper core/csrc/fps/fps_utils.py:6-21).
 * The two host-pointer symbols keep the reference's exact signature (blocking; they stage through the
 * GPU).  `farthest_point_sampling` (random start in the reference: srand(time(0)), :93-94) starts at
 * index `gdrn_fps_set_seed`-derived rand()%pn here; `_init_center` is deterministic and bit-exact.
 * ------------------------------------------------------------------------------------------- */
void farthest_point_sampling(float* pts, int* idxs, int pn, int sn);
void farthest_point_sampling_init_center(float* pts, int* idxs, int pn, int sn);
void gdrn_fps_set_seed(unsigned seed);
/* batched device version: pts [batch,pn,3] f32, idxs [batch,sn] i32.  start_idx: NULL -> bbox-centre
 * initialisation (init_center), else [batch] i32 explicit first index. */
int gdrn_fps_cuda(const float* pts, int* idxs, int pn, int sn, int batch, const int* start_idx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * PVNet RANSAC voting -- replaces core/csrc/ransac_voting/src/ransac_voting.cpp:30-109 (pybind module
 * `ransac_voting`: generate_hypothesis, voting_for_hypothesis, *_vanishing_point) and the kernels
 * src/ransac_voting_kernel.cu:11-49,88-126,170-229,268-310.
 *   direct [tn,vn,2] f32, coords [tn,2] f32, idxs [hn,vn,2] i32, hypo [hn,vn,2|3] f32 (pre-zeroed by the
 *   caller like at::zeros), inliers [hn,vn,tn] u8 (in/out, pre-zeroed by the caller).
 * ------------------------------------------------------------------------------------------- */
int rv_generate_hypothesis(const float* direct, const float* coords, const int* idxs, float* hypo, int tn, int vn,
                           int hn, void* stream);
int rv_voting_for_hypothesis(const float* direct, const float* coords, const float* hypo, unsigned char* inliers,
                             int tn, int vn, int hn, float inlier_thresh, void* stream);
int rv_generate_hypothesis_vanishing_point(const float* direct, const float* coords, const int* idxs, float* hypo,
                                           int tn, int vn, int hn, void* stream);
int rv_voting_for_hypothesis_vanishing_point(const float* direct, const float* coords, const float* hypo,
                                             unsigned char* inliers, int tn, int vn, int hn, float inlier_thresh,
                                             void* stream);
/* fused round: votes without materialising the [hn,vn,tn] mask; counts [hn,vn] i32 (overwritten). */
int rv_vote_count(const float* direct, const float* coords, const float* hypo, int* counts, int tn, int vn, int hn,
                  float inlier_thresh, int vanishing_point, void* stream);

/* The whole RANSAC voting layer for a batch of images on the device (SURVEY.md 8b "rv_ransac_round"): replaces the
 * Python driver ransac_voting_layer / ransac_voting_layer_v3 (core/csrc/ransac_voting/ransac_voting_gpu.py:7-104,
 * 123-218).  mask [b,h,w] f32 of non-negative integer weights (0 = background; a pixel of non-zero (int)weight is
 * one foreground pixel and adds its weight to the foreground count), vertex [b,h,w,vn,2] f32 -> win_pts [b,vn,2]:
 * ordered compaction of the foreground (tn stays on the device; images whose foreground count is below min_num give
 * zeros, above max_num keep each pixel with probability max_num / count), hn hypotheses per keypoint from pixel
 * pairs idxs [b,hn,vn,2] i32 (optional; taken modulo tn; NULL = counter-based RNG(seed)), fused vote + count,
 * per-keypoint winner, inlier set of the winner and least-squares refit of its lines.  No host synchronisation.  Optional outputs: hypo [b,hn,vn,2], counts
 * [b,hn,vn] i32, tn [b] i32, inliers [b,vn,h*w] u8 (compacted pixel order, first tn[b] entries valid). */
size_t rv_layer_workspace_bytes(int b, int h, int w, int vn, int hn);
int rv_ransac_voting_layer(const float* mask, const float* vertex, int b, int h, int w, int vn, int hn,
                           float inlier_thresh, int min_num, int max_num, unsigned seed, const int* idxs, float* win_pts,
                           float* hypo, int* counts, int* tn, unsigned char* inliers, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Chamfer / NN distance -- replaces core/csrc/torch_nndistance/src/nnd_cuda.cpp:37-84
 * (module torch_nndistance_aten: nnd_forward_cuda / nnd_backward_cuda; kernels nnd_cuda_kernel.cu:8-183).
 *   xyz1 [b,n,3], xyz2 [b,m,3] f32 -> dist1 [b,n], dist2 [b,m] f32, idx1 [b,n], idx2 [b,m] i32.
 *   backward: grad buffers are ACCUMULATED into (caller zeroes them, as torch_nndistance.py:52-53 does).
 * Returns 1 on success / 0 on failure like the reference launchers.
 * ------------------------------------------------------------------------------------------- */
int nnd_forward_cuda(const float* xyz1, const float* xyz2, float* dist1, float* dist2, int* idx1, int* idx2, int b,
                     int n, int m, void* stream);
int nnd_backward_cuda(const float* xyz1, const float* xyz2, float* gradxyz1, float* gradxyz2, const float* graddist1,
                      const float* graddist2, const int* idx1, const int* idx2, int b, int n, int m, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DeepIM depth-reprojection flow -- replaces core/csrc/flow/src/flow_cuda.cpp:30-42 (module flow_cuda,
 * kernel flow_cuda_kernel.cu:26-65). depth_src/tgt [B,1,H,W], KT [B,3,4], Kinv [B,3,3] ->
 * flow [B,2,H,W] (ch0 = dh, ch1 = dw), valid [B,1,H,W]; fp32.
 * ------------------------------------------------------------------------------------------- */
int flow_forward_cuda(const float* depth_src, const float* depth_tgt, const float* KT, const float* Kinv, float* flow,
                      float* valid, int batch, int height, int width, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Uncertainty PnP -- replaces core/csrc/uncertainty_pnp/src/uncertainty_pnp.cpp:61-92 (cffi surface
 * src/ext.h; Ceres AutoDiff + DENSE_SCHUR LM).  Host f64 pointers, blocking, same signature.
 * upnp_batched: device f64, `n_problems` independent problems of `pn` points each.
 * ------------------------------------------------------------------------------------------- */
void uncertainty_pnp(double* pts2d, double* pts3d, double* wgt2d, double* K, double* init_rt, double* result_rt,
                     int pn);
int upnp_batched(const double* pts2d, const double* pts3d, const double* wgt2d, const double* K,
                 const double* init_rt, double* result_rt, int pn, int n_problems, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Depth rasteriser -- replaces the GL renderers used for depth: lib/render_vispy/renderer.py:126-182,
 * 363-407 (Renderer.set_cam/draw_model/finish -> depth) and lib/egl_renderer/egl_renderer_v3.py:838-1228
 * (EGLRenderer.render(..., pc_cam_tensor=) -> pc_cam[...,2]); C++ side lib/egl_renderer/cpp/
 * egl_renderer.cpp:262-310.
 * Mesh registry (SURVEY.md 8b): rast_upload_mesh copies a mesh (verts [V,3] f32 in model space, metres; faces [F,3]
 * i32; host or device pointers) to the device once and returns its id (>= 0) or a negative error code.  The registry
 * is process-wide and append-only (at most 1024 meshes, all on the device current at the first upload): an id stays
 * valid for the life of the process, and the object that uploaded the mesh holds it.
 * rast_render_meshes renders n ROIs in one launch, ROI i with mesh mesh_ids[i] (i32, device) -- the multi-object form
 * of the reference's per-object draw_model loop (engine/gdrn_evaluator.py:520-526) without a host loop or a sync:
 *   poses [n,3,4] f32 (R|t, OpenCV camera), Ks [n,3,3] f32 -> depth [n,H,W] f32 (0 = background), optional
 *   xyz_cam [n,H,W,3]; zbuf_scratch of rast_scratch_bytes(n, H, W) bytes.
 *   quantize_bits: 0 = float depth of the interpolated camera-space z (EGL path), 24/16 = emulate the
 *   fixed-point z-buffer decode of the vispy path (renderer.py:176-182) with znear/zfar.
 * ------------------------------------------------------------------------------------------- */
int rast_upload_mesh(const float* verts, int V, const int* faces, int F);
/* rast_upload_mesh_ex: the same, with optional per-vertex colours [V,3] f32 in [0,1] (null: none), which
 * rast_render_meshes_rgb interpolates.  rast_upload_mesh(...) is rast_upload_mesh_ex(..., NULL). */
int rast_upload_mesh_ex(const float* verts, int V, const int* faces, int F, const float* colors);
int rast_mesh_count(void);
int rast_render_meshes(const int* mesh_ids, const float* poses, const float* Ks, int n, int H, int W, float znear,
                       float zfar, int quantize_bits, float* depth, float* xyz_cam, unsigned long long* zbuf_scratch,
                       void* stream);
size_t rast_scratch_bytes(int n, int H, int W);
/* rast_render_meshes_rgb: the same n renders in colour, with lib/pysixd/renderer_py.py's flat shading (light at the
 *   eye origin, ambient 0.5, face normal turned toward the viewer): rgb [n,H,W,3] u8 = rint(light_w * colour * 255),
 *   0 on background, and float-z depth [n,H,W] equal to rast_render_meshes(quantize_bits = 0).  Colour: colors [n,3]
 *   f32 per render when non-null, else the mesh's texture (rast_upload_mesh_tex: the nearest level-0 texel at the
 *   interpolated UV, clamp to edge -- renderer_py's texture2D), else its vertex colours (interpolated
 *   perspective-correctly), else grey 0.5.
 *   tri_ids [n,H,W] i32 (optional): the triangle seen at each pixel, -1 on background. */
int rast_render_meshes_rgb(const int* mesh_ids, const float* poses, const float* Ks, const float* colors, int n, int H,
                           int W, float znear, float zfar, uint8_t* rgb, float* depth, int* tri_ids,
                           unsigned long long* zbuf_scratch, void* stream);
/* rast_upload_mesh_tex: rast_upload_mesh_ex with optional shading attributes (null: none): normals [V,3] f32 (model
 *   space), uvs [V,2] f32 and texture [tex_h, tex_w, 3] u8 (row 0 at t = 0, i.e. the image already flipped as GL
 *   takes it; needs uvs).  The texture's mip chain (2x2 box filter, rounded) is built on the device here, once.
 *   rast_upload_mesh_ex(...) is rast_upload_mesh_tex(..., NULL, NULL, NULL, 0, 0). */
int rast_upload_mesh_tex(const float* verts, int V, const int* faces, int F, const float* colors, const float* normals,
                         const float* uvs, const uint8_t* texture, int tex_h, int tex_w);
/* rast_render_scene: the n_inst instances mesh_ids[i] (i32, device) at poses [n_inst,3,4] f32 rendered into ONE image
 *   with one z-buffer and one K [3,3] f32 -- the draw loop of lib/egl_renderer/egl_renderer_v3.py:998-1177 in one
 *   launch set.  A depth tie between instances goes to the earlier one.  light: HOST [12] f32 = light position (camera
 *   frame), light colour, material diffuse, material ambient.  depth [H,W] is required; every other output is written
 *   only when non-null: pc_cam [H,W,3] (== rast_render_meshes' xyz_cam), pc_obj [H,W,3] (model-space point), normal
 *   [H,W,3] (0.5 n + 0.5 of the interpolated camera-frame normal), image [H,W,3] (shader_textureless_texture.frag
 *   colour in [0,1], RGB), seg [H,W] (instance index + 1); all 0 on background.  scratch: rast_scene_scratch_bytes
 *   (n_inst, H, W) bytes, 8-aligned. */
int rast_render_scene(const int* mesh_ids, const float* poses, int n_inst, const float* K, int H, int W, float znear,
                      float zfar, const float* light, float* depth, float* pc_cam, float* pc_obj, float* normal,
                      float* image, float* seg, void* scratch, void* stream);
/* rast_render_scene_bg: rast_render_scene with an optional background [H,W,3] u8 (device; NULL: none).  Where no
 *   instance covers a pixel, image takes v / 255 in f32 per channel, in the background's channel order; every other
 *   output, and image on covered pixels, equals the render without a background.  n_inst may be 0 when a background is
 *   given (mesh_ids and poses may then be NULL).  rast_render_scene(...) is rast_render_scene_bg(..., NULL, ...). */
int rast_render_scene_bg(const int* mesh_ids, const float* poses, int n_inst, const float* K, int H, int W, float znear,
                         float zfar, const float* light, const uint8_t* background, float* depth, float* pc_cam,
                         float* pc_obj, float* normal, float* image, float* seg, void* scratch, void* stream);
size_t rast_scene_scratch_bytes(int n_inst, int H, int W);

/* ---------------------------------------------------------------------------------------------
 * Fast depth refinement -- replaces GDRN_Evaluator.process_depth_refine
 * (core/gdrn_modeling/engine/gdrn_evaluator.py:521-561) == GdrnPredictor.process_depth_refine
 * (core/gdrn_modeling/demo/predictor_gdrn.py:239-286), one iteration after a render:
 *   xyz [n,3,hw,hw], mask [n,hw,hw], depth_sensor [n,hw,hw], ren_depth [n,hw,hw], K_crop [n,3,3],
 *   trans [n,3] in/out; thresh = DEPTH_REFINE_THRESHOLD (0.8); 0 < hw <= 128.
 *   mask_mode: get_out_mask (engine/engine_utils.py:313-333) folded into the kernel: 0 = `mask` is already
 *   normalised, 1 = raw L1 mask output -> per-ROI min-max normalisation, 2 = raw logits -> sigmoid.
 *   weight_mode: 0 = ||xyz||, 1 = TEST.USE_COOR_Z_REFINE (gdrn_evaluator.py:528-537): w = (R xyz)_z * mask *
 *   (ren > 0) * (sensor > 0) with `xyz` the raw [0,1] coordinate maps and rot [n,3,3] the rotation of the pose being
 *   refined (may be NULL for mode 0).  Signed weights follow the reference's order: divide by the sum, then threshold
 *   against the max over all pixels; a zero sum leaves t unchanged.  So does an empty selection (a constant L1
 *   mask, thresh >= 1), where the reference's median of nothing is NaN.  Sums below 2^-128 in magnitude are
 *   normalised without overflowing the f32 reciprocal (INTEGRATION.md section 7).
 * ------------------------------------------------------------------------------------------- */
int gdrn_depth_refine_step(const float* xyz, const float* mask, int mask_mode, const float* depth_sensor,
                           const float* ren_depth, const float* K_crop, const float* rot, int weight_mode, float* trans,
                           int n, int hw, float thresh, void* stream);
/* gdrn_depth_refine_trace: the same kernel and output (trans bit-identical to gdrn_depth_refine_step), plus a record
 * of every stage.  Trace buffers (device, all required; the caller initialises them, entries a ROI does not reach --
 * after a zero sum, or with nothing selected -- keep that value):
 *   tr_m_lo, tr_m_scale [n] f32 the mask normalisation (m - m_lo) / m_scale (0 and 1 unless mask_mode 1);
 *   tr_w [n,hw*hw] f32 raw weights; tr_sum [n] f64; tr_max, tr_min [n] f32 (zero included); tr_cut [n] f32;
 *   tr_sel [n,hw*hw] u8 selected pixels; tr_count [n] i32; tr_median [n] f32; tr_centroid [n,2] f64 (y, x);
 *   tr_ray [n,3] f64 K^-1 (x, y, 1) / z; tr_t [n,3] f32 the output translation. */
int gdrn_depth_refine_trace(const float* xyz, const float* mask, int mask_mode, const float* depth_sensor,
                            const float* ren_depth, const float* K_crop, const float* rot, int weight_mode, float* trans,
                            int n, int hw, float thresh, float* tr_m_lo, float* tr_m_scale, float* tr_w, double* tr_sum,
                            float* tr_max, float* tr_min, float* tr_cut, unsigned char* tr_sel, int* tr_count,
                            float* tr_median, double* tr_centroid, double* tr_ray, float* tr_t, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ROI crop + resize (SURVEY.md 8f rank 1) -- replaces crop_resize_by_warp_affine = cv2.warpAffine
 * (core/utils/data_utils.py:115-133) as called once per ROI by GdrnPredictor.preprocessing
 * (core/gdrn_modeling/demo/predictor_gdrn.py:417-438) and the test data loader
 * (core/gdrn_modeling/datasets/data_loader.py:758-797).  OpenCV's warpAffine arithmetic is reproduced exactly
 * (bit-exact for uint8 and nearest, bit-exact with the scalar float path for float bilinear; zero border).
 *   M [n,6] f64 (device): forward (source -> crop) 2x3 matrices, row-major, as get_affine_transform returns them.
 *   gdrn_crop_resize_u8 : image [H,W,C] u8 (BGR as cv2.imread, device), INTER_LINEAR, followed by
 *                         normalize_image ((v - pixel_mean[c]) / pixel_std[c] in f64 -> f32; host arrays [C])
 *                         -> out [n,C,out_h,out_w] f32 (the roi_img the model consumes).
 *   gdrn_crop_resize_f32: src [H,W,C] f32 (device), INTER_LINEAR (nearest = 0; roi_coord_2d) or INTER_NEAREST
 *                         (nearest = 1; roi_depth) -> out [n,C,out_h,out_w] f32.
 * ------------------------------------------------------------------------------------------- */
int gdrn_crop_resize_u8(const uint8_t* image, int H, int W, int C, const double* M, int n, int out_h, int out_w,
                        const double* pixel_mean, const double* pixel_std, float* out, void* stream);
int gdrn_crop_resize_f32(const float* src, int H, int W, int C, const double* M, int n, int out_h, int out_w,
                         int nearest, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Model inputs for the ROIs of many images in one forward -- replaces the per-image read_data_test
 * (core/gdrn_modeling/datasets/data_loader.py:751-797) + batch_data_test (engine/engine_utils.py:213-241) of the
 * reference's test loop (build_gdrn_test_loader, batch_size = 1).
 *
 * gdrn_roi_setup: one thread per ROI, the loader's dtype path step for step (see csrc/roi_batch.cu).
 *   det_meta [n,2] i32 (image index, label), det_xywh [n,4] f32 (bbox_est, XYWH_ABS); per image K [N,3,3] f32 and
 *   im_hw [N,2] i32 (H, W); extents [nc,3] f32 per label.  Outputs with batch_data_test's dtypes: roi_center [n,2],
 *   roi_wh [n,2], scale [n], resize_ratio [n], roi_extent [n,3], roi_cam [n,3,3], im_H [n], im_W [n], bbox_xyxy [n,4]
 *   (f32), roi_cls [n] (i64), and the forward affine matrices M_in / M_out [n,6] f64 of get_affine_transform for
 *   in_res / out_res.  Indices are not range-checked on the device: the caller validates them.
 * gdrn_roi_crop_multi: every crop of the batch in one launch, with crop_resize.cu's exact warpAffine arithmetic;
 *   ROI i reads image det_meta[i].image.
 *   images [N,H,W,C] u8 BGR, C = 1 (replicated to three channels, as cv2.imread(..., IMREAD_COLOR)) or 3;
 *   pixel_mean / pixel_std: host arrays [3].
 *   -> roi_img [n,3,in_res,in_res] f32 (bilinear + normalize_image);
 *      roi_coord_2d [n,2,out_res,out_res] f32: bilinear crop of get_2d_coord_np's grid, computed in the kernel;
 *   optional (NULL to skip; they need depth [N,H,W] u16 and depth_factor [N] f64, device):
 *      roi_depth [n,1,in_res,in_res] f32: nearest crop of f32((double)depth / depth_factor) metres;
 *      depth_sensor [n,out_res,out_res] f32: ((a+b)+(c+d))*0.25 of the centre 2x2 of every 4x4 cell of roi_depth
 *      (in_res = 4 * out_res), the sensor crop depth refine reads.
 * ------------------------------------------------------------------------------------------- */
int gdrn_roi_setup(const int* det_meta, const float* det_xywh, int n, const float* K, const int* im_hw,
                   const float* extents, double dzi_pad_scale, int in_res, int out_res, float* roi_center, float* roi_wh,
                   float* scale, float* resize_ratio, float* roi_extent, float* roi_cam, long long* roi_cls, float* im_H,
                   float* im_W, float* bbox_xyxy, double* M_in, double* M_out, void* stream);
int gdrn_roi_crop_multi(const uint8_t* images, int H, int W, int C, const int* det_meta, const double* M_in,
                        const double* M_out, int n, int in_res, int out_res, const double* pixel_mean,
                        const double* pixel_std, const uint16_t* depth, const double* depth_factor, float* roi_img,
                        float* roi_coord_2d, float* roi_depth, float* depth_sensor, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched RANSAC-PnP (SURVEY.md 8f rank 2) -- replaces the per-ROI host loop get_pnp_ransac_pose
 * (core/gdrn_modeling/engine/gdrn_evaluator.py:1122-1221) + misc.pnp_v2 (lib/pysixd/misc.py:153-208) =
 * cv2.solvePnPRansac(EPNP, reprojectionError 3, 100 iterations), the reference predictor's default TEST.USE_PNP path.
 * One CTA per ROI: correspondence selection from the maps, `iters` P3P hypotheses, inlier counts, LM refit on the
 * inliers (csrc/pnp_ransac.cu).  poses [n,3,4] (R|t, -100 everywhere when fewer than 4 correspondences / no model),
 * n_inliers [n] (optional), inlier_mask [n, hw*hw | npts] u8 over the INPUT pixels / points (optional).
 * idxs (optional) [n, iters, 4] i32: the sampled correspondences of every hypothesis (taken modulo the number of
 * selected correspondences) instead of the built-in counter-based RNG(seed).
 *   _maps  : coor_x/y/z, mask [n, hw, hw] raw network outputs, roi_coord_2d [n,2,hw,hw], im_hw [n,2] = (im_H, im_W),
 *            extents [n,3], Ks [n,3,3]; mask_thr = GEO_HEAD.MASK_THR_TEST (0.5).
 *   _points: explicit correspondences pts3d [n,npts,3], pts2d [n,npts,2] (all used), npts <= 4096.
 * ------------------------------------------------------------------------------------------- */
int gdrn_pnp_ransac_maps(const float* coor_x, const float* coor_y, const float* coor_z, const float* mask,
                         const float* roi_coord_2d, const float* im_hw, const float* extents, const float* Ks,
                         const int* idxs, int n, int hw, int iters, float mask_thr, float reproj_thr, unsigned seed,
                         float* poses, int* n_inliers, unsigned char* inlier_mask, void* stream);
int gdrn_pnp_ransac_points(const float* pts3d, const float* pts2d, const float* Ks, const int* idxs, int n, int npts,
                           int iters, float reproj_thr, unsigned seed, float* poses, int* n_inliers,
                           unsigned char* inlier_mask, void* stream);
/* gdrn_pnp_ransac_trace: the same kernel and outputs (bit-identical to the two entries above), plus a record of every
 * stage.  Maps form when pts3d is null (npts = hw*hw), points form otherwise (the map arguments are then ignored).
 * Trace buffers (device, all required; the caller initialises them, entries a ROI does not reach keep that value):
 *   tr_count [n] i32 selected correspondences N; tr_src [n,4096] i32 source pixel / point of compacted entry i (-1 from N);
 *   tr_samples [n,iters,4] i32 the ids each hypothesis used (after % N and de-duplication); tr_nsol [n,iters] i32 P3P
 *   solutions; tr_hyp [n,iters,12] f64 the solution chosen by the fourth point; tr_cnt [n,iters] i32 inlier count
 *   (-1 no model); tr_best [n] i32; tr_inl [n,2,4096] u8 inlier flags at the start of each refit round (compacted
 *   order); tr_round_pose [n,2,2,12] f64 start / end pose of each round; tr_round_cost [n,2,3] f64 cost at the start,
 *   the lowest cost the LM evaluated and the cost at the returned pose; tr_pose [n,12] f64 final pose (-100 for the
 *   sentinel). */
int gdrn_pnp_ransac_trace(const float* coor_x, const float* coor_y, const float* coor_z, const float* mask,
                          const float* roi_coord_2d, const float* im_hw, const float* extents, const float* pts3d,
                          const float* pts2d, const float* Ks, const int* idxs, int n, int npts, int iters,
                          float mask_thr, float reproj_thr, unsigned seed, float* poses, int* n_inliers,
                          unsigned char* inlier_mask, int* tr_count, int* tr_src, int* tr_samples, int* tr_nsol,
                          double* tr_hyp, int* tr_cnt, int* tr_best, unsigned char* tr_inl, double* tr_round_pose,
                          double* tr_round_cost, double* tr_pose, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Network-initialised PnP (TEST.PNP_TYPE = net_*) -- replaces the per-ROI host loop process_net_and_pnp
 * (core/gdrn_modeling/engine/gdrn_evaluator.py:241-371).  Same correspondences as gdrn_pnp_ransac_maps; rot_net [n,3,3]
 * and trans_net [n,3] are the network's pose.  pnp_type:
 *   0 net_iter_pnp       cv2.solvePnP(ITERATIVE, useExtrinsicGuess): LM over all correspondences from the network pose
 *                        (at most 20 iterations).  The reference's 1 m translation guard never fires for this type
 *                        (cv2 writes the result into the guess it is compared with), so none is applied.
 *   1 net_ransac_pnp     RANSAC at `ransac_iters` (the reference passes 20); ||t - t_net|| > 1 m -> t = t_net.
 *   2 net_ransac_pnp_rot R from the RANSAC step, t = t_net.
 * < 4 correspondences, or no RANSAC model -> the network pose.  n_used [n] (optional): the correspondences the pose was
 * fitted to (all selected ones for 0, the inliers for 1 / 2), 0 where the network pose is returned.  No host sync.
 * gdrn_pnp_iterative_points: type 0 on explicit correspondences pts3d [n,npts,3], pts2d [n,npts,2] from (rot0, trans0).
 * ------------------------------------------------------------------------------------------- */
int gdrn_pnp_net_maps(const float* coor_x, const float* coor_y, const float* coor_z, const float* mask,
                      const float* roi_coord_2d, const float* im_hw, const float* extents, const float* Ks,
                      const float* rot_net, const float* trans_net, int n, int hw, int pnp_type, float mask_thr,
                      float reproj_thr, int ransac_iters, unsigned seed, float* poses, int* n_used, void* stream);
int gdrn_pnp_iterative_points(const float* pts3d, const float* pts2d, const float* Ks, const float* rot0,
                              const float* trans0, int n, int npts, float* poses, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Online training targets (SURVEY.md 8f rank 3) -- after rast_render_meshes, replaces the torch ops of
 * core/gdrn_modeling/engine/engine_utils.py:131-187: misc.calc_xyz_bp_batch (lib/pysixd/misc.py:412-457),
 * roi_mask_obj, xyz_to_region_batch (core/utils/data_utils.py:283-301) and the xyz normalisation, in one kernel.
 *   depth [n,H,W], R [n,3,3] (ego rotation), T [n,3], K [n,3,3] (zoomed intrinsics), fps_points [n,F,3], extents [n,3]
 *   -> roi_xyz [n,3,H,W] (xyz / extent + 0.5), xyz_raw [n,H,W,3] (object-space xyz), mask_obj [n,H,W] f32,
 *      region [n,H,W] i64 (1..F, 0 = background).  Any output may be NULL.
 * ------------------------------------------------------------------------------------------- */
int gdrn_xyz_region_targets(const float* depth, const float* R, const float* T, const float* K, const float* fps_points,
                            const float* extents, int n, int H, int W, int F, float* roi_xyz, float* xyz_raw,
                            float* mask_obj, long long* region, void* stream);

/* ---------------------------------------------------------------------------------------------
 * YOLOX head post-processing (SURVEY.md 8f rank 4) -- replaces YOLOXHead.decode_outputs
 * (det/yolox/models/yolo_head.py:239-255) and postprocess (det/yolox/utils/boxes.py:34-80: cxcywh -> xyxy, class
 * max, obj * cls_conf >= conf_thre, torchvision batched_nms / nms) for a batch of images, no host synchronisation.
 *   preds [B, A, 5 + num_classes] f32 (obj / class scores already sigmoid-ed like the head emits them);
 *   n_levels > 0: raw head outputs, decoded here with hw [n_levels,2] i32 (rows, cols per level) and strides [n_levels]
 *   i32 (both device arrays); n_levels = 0: preds are already decoded (cx, cy, w, h).
 *   dets [B, max_out, 7] = (x1, y1, x2, y2, obj_conf, class_conf, class) in descending score order, n_det [B] i32.
 *   The NMS decides as torchvision on CUDA does (sm_90 build): class-aware with n <= 25 000 candidates in an image
 *   (boxes.numel() <= 100 000) is _batched_nms_coordinate_trick -- boxes shifted by cls * (max coordinate + 1) in fp32,
 *   every pair compared; above that _batched_nms_vanilla -- per class, unshifted; class-agnostic is nms.  IoU as
 *   nms_kernel_impl<float>: fma(bw, bh, Sa) - inter in the denominator (b the later-ranked box), IoU > nms_thre.
 *   yolox_postprocess_layout: offsets[6] = byte offsets, from the workspace rounded up to 256 bytes, of the stage
 *   results a call leaves there: cand [B,A,7] f32 (the compacted decoded rows), score [B,A] f32, order [B,A] i32
 *   (candidate index by rank), n_cand [B] i32, max_coord [B] f32, mask [B,A,(A+63)/64] u64 (words jb >= ib written).
 * ------------------------------------------------------------------------------------------- */
size_t yolox_postprocess_workspace_bytes(int B, int A);
int yolox_postprocess_layout(int B, int A, size_t* offsets);
int yolox_postprocess(const float* preds, int B, int A, int num_classes, const int* hw, const int* strides, int n_levels,
                      float conf_thre, float nms_thre, int class_agnostic, int max_out, float* dets, int* n_det,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pose outlines over a test image (csrc/vis_poses.cu), the per-dataset vis_poses_full scripts' pixel work for N images
 * of one size H x W.  No allocation, no synchronisation, the caller's stream.
 *   gdrn_vis_gray3: img [N,H,W,3] u8, B, G, R (or R, G, B with rgb_order = 1) -> out [N,H,W,3] u8, each channel
 *     (3735 b + 19235 g + 9798 r + 16384) >> 15, which is cv2.cvtColor(COLOR_BGR2GRAY) bit for bit.
 *   gdrn_vis_outlines: shaded [N,H,W,3] f32, the RGB image output of rast_render_scene_bg (background included), and
 *     cover [n,H,W] f32 (covered where != 0, e.g. rast_render_meshes depth) of the n GT and estimate instances;
 *     image j owns instances [inst_off[j], inst_off[j+1]) (inst_off [N+1] i32, device), is_gt [n] u8 (device) flags
 *     the GT ones.  An instance's edge pixel is covered with an uncovered pixel exactly bw rows or columns away in one
 *     of the four directions (a neighbour outside the image does not count).  -> out [N,H,W,3] u8 BGR: (0, 255, 0)
 *     on any estimate edge, else (255, 0, 0) on any GT edge, else (u8)(shaded[2 - c] * 255 + 0.5) in f32 without
 *     contraction (to_bgr, to_255, then + 0.5 truncated). */
int gdrn_vis_gray3(const uint8_t* img, int N, int H, int W, int rgb_order, uint8_t* out, void* stream);
int gdrn_vis_outlines(const float* shaded, const float* cover, const int* inst_off, const uint8_t* is_gt, int N, int n,
                      int H, int W, int bw, uint8_t* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * YOLOX training loss (csrc/yolox_loss.cu) -- replaces YOLOXHead.get_losses (det/yolox/models/yolo_head.py:256-426):
 * SimOTA assignment and the IoU, objectness, class and L1 terms for a batch, no host synchronisation (DESIGN.md §7q).
 *   outputs [B, A, 5 + num_classes] (decoded cx, cy, w, h; objectness and class logits) and origin_preds [B, A, 4] (raw
 *   regression; may be NULL when use_l1 = 0), both of dtype 0 = f32, 1 = f16, 2 = bf16; labels [B, M, 5] f32 (class,
 *   cx, cy, w, h; the GTs of an image are its first n rows, n = rows with a positive sum; M <= 1024); shifts [3, A] f32 =
 *   x shift, y shift, stride per anchor.  Everything is computed in f32.
 *   yolox_loss_forward: trace (NULL or [B, M, A, 3] f32) receives (IoU, unpenalised cost, cost) of every candidate pair.
 *   yolox_loss_backward: grad_losses [4] f32 (device) = upstream gradients of loss_iou (already x5), loss_conf,
 *   loss_cls, loss_l1; reads the assignment the forward left in the same workspace; grad_outputs like outputs,
 *   grad_origin like origin_preds (written when use_l1).
 *   yolox_loss_layout: offsets[16] = byte offsets, from the workspace rounded up to 256 bytes, of nlabel [B] i32,
 *   cand [B,A] u8, cls_sum [B,A] f32, count [B,A] i32, chooser [B,A] i32, n_cand [B] i32, k [B,M] i32, iou_sum [B,M]
 *   f32, chosen [B,M,10] i32 (-1 padded), fg [B,A] u8, matched [B,A] i32, iou_t [B,A] f32, partial [P,4] f32,
 *   partial_fg [P] i32, err [B] i32 and result [8] f32 = loss_iou * 5, loss_conf, loss_cls, loss_l1, max(num_fg, 1),
 *   num_fg / max(num_gt, 1), class-id error flag, num_fg.
 * ------------------------------------------------------------------------------------------- */
size_t yolox_loss_workspace_bytes(int B, int A, int M);
int yolox_loss_layout(int B, int A, int M, size_t* offsets);
int yolox_loss_forward(const void* outputs, const void* origin_preds, int dtype, const float* labels, const float* shifts,
                       int B, int A, int num_classes, int M, int use_l1, float* trace, void* workspace,
                       size_t workspace_bytes, void* stream);
int yolox_loss_backward(const void* outputs, const void* origin_preds, int dtype, const float* labels, const float* shifts,
                        int B, int A, int num_classes, int M, int use_l1, const float* grad_losses, void* workspace,
                        size_t workspace_bytes, void* grad_outputs, void* grad_origin, void* stream);

/* ---------------------------------------------------------------------------------------------
 * GDRN training loss (csrc/gdrn_loss.cu) -- replaces GDRN_DoubleMask.gdrn_loss
 * (core/gdrn_modeling/models/GDRN_double_mask.py:287-536) with PyPMLoss and get_closest_rot_batch: the coordinate,
 * mask, full-mask and region terms, symmetry-aware point matching (PM_R_ONLY) and the centroid / z terms, all f32, no
 * host synchronisation (DESIGN.md §7r).
 *   inputs[22] (device pointers, NULL where a term is off): out_x, out_y, out_z, out_mask_vis, out_mask_full [B,1,H,W]
 *   (plane contiguous, batch strides in batch_strides[5], in elements); the GT masks the config selects for xyz, mask,
 *   full mask and region [B,H,W]; gt_xyz [B,3,H,W]; out_region [B,R1,H,W]; gt_region [B,H,W] i64; out_rot, gt_rot
 *   [B,3,3]; points [B,N,3]; extents [B,3]; symmetry table [T,3,3] and per-ROI (first row, count) [B,2] i32 (both NULL:
 *   no symmetry); out_centroid [B,2]; out_trans_z [B]; gt_trans_ratio [B,3]; gt_trans [B,3].  HW = H * W.
 *   weights[7] = XYZ_LW, MASK_LW, FULL_MASK_LW, REGION_LW, PM_LW, CENTROID_LW, Z_LW.  flags: 1 geometry terms (xyz,
 *   mask, region), 2 full mask, 4 mask BCE (else L1), 8 full mask BCE, 16 point matching, 32 PM_NORM_BY_EXTENT,
 *   64 centroid, 128 z, 256 Z_TYPE ABS (else REL).
 *   gdrn_loss_backward: grad_losses [9] f32 (device) = upstream gradients of the result's losses; grads[9] = device
 *   outputs for out_x, out_y, out_z, out_mask_vis, out_mask_full [B,HW], out_region [B,R1,HW], out_rot [B,9],
 *   out_centroid [B,2], out_trans_z [B] (NULL where a term is off); reads what the forward left in the workspace.
 *   gdrn_loss_layout: offsets[10] = byte offsets, from the workspace rounded up to 256 bytes, of partial [P,8] f64
 *   (per CTA: |dx|, |dy|, |dz|, mask, full mask and region CE sums, xyz and region mask counts; P = B * ceil(HW / 512)),
 *   partial_err [P] i32, lse [B,HW] f32, sym_idx [B] i32 (-1 = R_gt, k = R_gt S_k), rot_sel [B,3,3] f32 (R_gt'),
 *   pm_abs [B] f64, pm_sign [B,3,3] f64 (sum of sign(w (R_est - R_gt') p)_i w p_j), sym_err [B] f32 (degrees),
 *   norm [4] f32 (xyz count, region count, each at least 1; B * HW; B * N * 3) and result [10] f32 = loss_coor_x / y /
 *   z, loss_mask, loss_mask_full, loss_region, loss_PM_R, loss_centroid, loss_z (each times its weight), region-label
 *   error flag.
 * ------------------------------------------------------------------------------------------- */
size_t gdrn_loss_workspace_bytes(int B, int HW);
int gdrn_loss_layout(int B, int HW, size_t* offsets);
int gdrn_loss_forward(const void* const* inputs, const long long* batch_strides, const float* weights, int B, int HW,
                      int R1, int N, int flags, void* workspace, size_t workspace_bytes, void* stream);
int gdrn_loss_backward(const void* const* inputs, const long long* batch_strides, const float* weights, int B, int HW,
                       int R1, int N, int flags, const float* grad_losses, void* const* grads, void* workspace,
                       size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * YOLOX detector network (det/yolox/models: CSPDarknet + YOLOPAFPN + YOLOXHead, inference), csrc/yolox_net.cu.
 *   yolox_model_create: one engine per (depth, width, num_classes, max_batch, H, W, precision); H, W multiples of 32;
 *     precision 1 = bf16x3 (split-bf16 operands), 0 = bf16.  Channel counts must be multiples of 8.
 *   yolox_model_load_tensor: one tensor of a reference state dict by name (device f32, numel elements): unfused
 *     (conv.weight + bn.weight / bias / running_mean / running_var, BatchNorm eps 1e-3) or fused (conv.weight +
 *     conv.bias); prediction convs as head.{cls,reg,obj}_preds.k.{weight,bias}.  Synchronises the stream (load time).
 *   yolox_model_missing: folds BatchNorm in float64 and packs every conv whose tensors are all present; returns how
 *     many convs still lack a tensor (0 = ready).
 *   yolox_model_workspace_bytes(B): caller-owned activation workspace for a forward of B images (chunks of max_batch).
 *   yolox_model_forward: img [B,3,H,W] f32 (BGR, 0..255) -> det_preds [B, A, 5 + num_classes] f32 (decoded boxes
 *     cx, cy, w, h; sigmoid obj; sigmoid classes), A = yolox_model_num_anchors.  No allocation, no synchronisation.
 *   yolox_model_set_scales: multi-scale test-time augmentation (YOLOX.forward(augment=True), model_utils.scale_img):
 *     one layer plan per scale s over the same packed weights, for the create-time H x W resampled (bilinear,
 *     align_corners=False) to (int)(H*s) x (int)(W*s) and padded with 0.447*255 to ceil(H*s/32)*32 x ceil(W*s/32)*32;
 *     s == 1.0 is the plain plan.  Replaces the previous set.  Host only, no CUDA call; a scale with an empty resampled
 *     image is an error.
 *   yolox_model_num_anchors_tta: A_tta, the anchors summed over the scales.
 *   yolox_model_workspace_bytes_tta(B): workspace of yolox_model_forward_tta (the largest plan's).
 *   yolox_model_forward_tta: img [B,3,H,W] -> det_preds [B, A_tta, 5 + num_classes], the scales' outputs in scale order
 *     along the anchor axis, boxes of scale s multiplied by 1.0f / (float)s (torch's det[..., :4] /= s on CUDA).  Scales
 *     run one after the other per max_batch chunk in one workspace.  No allocation, no synchronisation.
 *   yolox_postprocess_single: keep-single-instance post-process of the reference predictor (predictor_yolo.py:84-140):
 *     per class the highest-scoring anchor with obj * cls_conf >= conf_thre, class-agnostic NMS, rows in ascending
 *     class order; dets [B, num_classes, 7], n_det [B] i32.  Classes without such an anchor are left out.  The
 *     reference runs this NMS with torchvision's CPU nms: products rounded one by one, and the fp32 IoU compared with
 *     nms_thre as a double (so a threshold that rounds up in fp32, such as 0.3, is honoured); num_classes <= 1024.
 *   yolox_postprocess_single_layout: offsets[3] = byte offsets, from the workspace rounded up to 256 bytes, of score
 *     [B,A] f32, cls [B,A] i32 and sel [B,num_classes] i32 (selected anchor per class, -1 = none) a call leaves there.
 * ------------------------------------------------------------------------------------------- */
typedef struct YoloxModel YoloxModel;
int yolox_model_create(YoloxModel** out, double depth, double width, int num_classes, int max_batch, int H, int W, int precision);
void yolox_model_destroy(YoloxModel* m);
int yolox_model_load_tensor(YoloxModel* m, const char* key, const float* data, int64_t numel, void* stream);
int yolox_model_missing(YoloxModel* m);
int yolox_model_num_anchors(const YoloxModel* m);
size_t yolox_model_workspace_bytes(YoloxModel* m, int B);
int yolox_model_forward(YoloxModel* m, const float* img, int B, float* det_preds, void* workspace, size_t workspace_bytes,
                        void* stream);
int yolox_model_set_scales(YoloxModel* m, const double* scales, int n_scales);
int yolox_model_num_anchors_tta(const YoloxModel* m);
size_t yolox_model_workspace_bytes_tta(YoloxModel* m, int B);
int yolox_model_forward_tta(YoloxModel* m, const float* img, int B, float* det_preds, void* workspace, size_t workspace_bytes,
                            void* stream);
size_t yolox_postprocess_single_workspace_bytes(int B, int A, int num_classes);
int yolox_postprocess_single_layout(int B, int A, int num_classes, size_t* offsets);
int yolox_postprocess_single(const float* preds, int B, int A, int num_classes, float conf_thre, double nms_thre, float* dets,
                             int* n_det, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * BOP pose errors over a batch of P (estimate, GT) pairs -- replaces the per-pair numpy loops of lib/pysixd/pose_error.py
 * (vsd, mssd, mspd, add, adi) as eval_calc_errors.py drives them.  Results do not depend on the launch shape.
 *
 * gdrn_vsd_errors: depth_est [Ne,H,W], depth_gt [Ng,H,W] (rendered camera-space z), depth_test [Ni,H,W] (0 = missing),
 *   all f32; pair p reads images pair_est[p], pair_gt[p], pair_img[p] (i32); Ks [P,3,3] f64, diameters [P] f64,
 *   gate [P] u8 (0 = sphere projections do not overlap -> 1.0 for every tau); taus [T] f64 (T <= 32); delta is compared
 *   in f32 as the reference does.  errors [P,T] f64 equal the reference's numpy vsd (bop19 visibility, step cost) bit
 *   for bit.  counts_ws: gdrn_vsd_workspace_bytes(P, T) bytes of 64-bit pixel counts (zeroed here).
 * gdrn_sym_max_dist: pts [sum N_o, 3] f64 with pt_offsets [O+1] i64; syms [sum S_o, 3, 4] f64 ([R|t]) with sym_offsets
 *   [O+1] i64 (S_o >= 1); pair_obj [P] i32 indexes the objects; pose_est / pose_gt [P,3,4] f64, Ks [P,3,3] f64;
 *   max_syms = max S_o.  mssd [P] (inf where gate_mssd[p] == 0) and mspd [P] in the units of pts / pixels.
 * gdrn_ad_errors: use_adi [P] u8 picks ADI (1) or ADD (0); gate [P] u8 (0 -> inf); max_pts = max N_o;
 *   ws: gdrn_ad_workspace_bytes(P, max_pts) bytes.  err [P] f64.
 * gdrn_sym_proj_mean: pts, syms, pair_obj, poses and Ks as gdrn_sym_max_dist; use_syms [P] u8 picks the object's
 *   symmetry set (1, arp_2d_sym / projS) or the GT pose alone (0, arp_2d / proj; the set of an object with a continuous
 *   symmetry holds no identity).  err [P] f64 = min over the symmetries of the mean pixel distance, points projected as
 *   transform_pts_Rt_2d does (camera space, then K, then / z); max_syms = max over pairs of S_o (or 1).
 * gdrn_sym_rt_errors: syms, pair_obj, poses and use_syms as above; re_deg [P] f64 = re / re_sym in degrees, te [P] f64 =
 *   te / te_sym in the units of t, each minimised over the symmetries on its own.
 * ------------------------------------------------------------------------------------------- */
size_t gdrn_vsd_workspace_bytes(int P, int T);
int gdrn_vsd_errors(const float* depth_est, const float* depth_gt, const float* depth_test, int H, int W,
                    const int* pair_est, const int* pair_gt, const int* pair_img, const double* Ks, const double* diameters,
                    const uint8_t* gate, int P, const double* taus, int T, float delta, int normalized_by_diameter,
                    void* counts_ws, size_t ws_bytes, double* errors, void* stream);
int gdrn_sym_max_dist(const double* pts, const int64_t* pt_offsets, const double* syms, const int64_t* sym_offsets,
                      const int* pair_obj, const double* pose_est, const double* pose_gt, const double* Ks,
                      const uint8_t* gate_mssd, int P, int max_syms, double* mssd, double* mspd, void* stream);
size_t gdrn_ad_workspace_bytes(int P, int max_pts);
int gdrn_ad_errors(const double* pts, const int64_t* pt_offsets, const int* pair_obj, const double* pose_est,
                   const double* pose_gt, const uint8_t* use_adi, const uint8_t* gate, int P, int max_pts, void* ws,
                   size_t ws_bytes, double* err, void* stream);
int gdrn_sym_proj_mean(const double* pts, const int64_t* pt_offsets, const double* syms, const int64_t* sym_offsets,
                       const int* pair_obj, const double* pose_est, const double* pose_gt, const double* Ks,
                       const uint8_t* use_syms, int P, int max_syms, double* err, void* stream);
int gdrn_sym_rt_errors(const double* syms, const int64_t* sym_offsets, const int* pair_obj, const double* pose_est,
                       const double* pose_gt, const uint8_t* use_syms, int P, double* re_deg, double* te, void* stream);

/* ---------------------------------------------------------------------------------------------
 * YOLOX test-time letterbox (csrc/yolox_letterbox.cu): N uint8 HWC images of one size (C = 1 is replicated to BGR)
 * -> out [N,3,th,tw] f32, the image resized to (int(h r), int(w r)) with r = min(th/h, tw/w), bit-exact to
 * cv2.resize(INTER_LINEAR), placed top-left on a 114 canvas.  When ValTransform's second resize is not the identity for
 * that size the image is resized twice through a u8 workspace of yolox_letterbox_workspace_bytes (0 otherwise).
 * ------------------------------------------------------------------------------------------- */
size_t yolox_letterbox_workspace_bytes(int N, int H, int W, int th, int tw);
int yolox_letterbox(const uint8_t* images, int N, int H, int W, int C, int th, int tw, float* out, void* workspace,
                    size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * COCO bbox evaluation (csrc/coco_eval.cu), pycocotools COCOeval evaluate + accumulate.  P (image, category) pairs in
 * (category, image) order; GT and detections grouped by pair (input order kept inside a pair), offsets [P+1].
 *   coco_eval_match: per pair the kept detections (stable descending score, at most max_det; kept offsets
 *     pair_kept_off [P+1], Dkept in all) -> dt_order (input index), kept_score, kept_rank; ious at pair_iou_off
 *     (kept x G per pair); gt_ignore [A,Gtot]; dt_match [A,T,Dkept] (matched GT index + 1, 0 = none);
 *     dt_ignore [A,T,Dkept]; gt_match [A,T,Gtot] (kept position + 1 of the matching detection, 0 = none).
 *   coco_eval_accumulate: per category (cat_off [K+1] over kept detections, cat_gt_off [K+1] over GT, cat_pairs [K])
 *     precision [T,R,K,A,M] and recall [T,K,A,M], both pre-filled with -1 by the caller.
 * ------------------------------------------------------------------------------------------- */
int coco_eval_match(const double* gt_box, const double* gt_area, const uint8_t* gt_crowd, const double* dt_box,
                    const double* dt_score, const int* pair_gt_off, const int* pair_dt_off, const int* pair_kept_off,
                    const long long* pair_iou_off, int P, int Gtot, int Dkept, const double* iou_thrs, int T,
                    const double* area_rng, int A, int max_det, int* dt_order, double* kept_score, int* kept_rank,
                    double* ious, uint8_t* gt_ignore, int* dt_match, uint8_t* dt_ignore, int* gt_match, void* stream);
size_t coco_eval_accumulate_workspace_bytes(int Dkept);
int coco_eval_accumulate(const double* kept_score, const int* kept_rank, const int* dt_match, const uint8_t* dt_ignore,
                         const uint8_t* gt_ignore, const int* cat_off, const int* cat_gt_off, const int* cat_pairs,
                         int max_cat_dets, int K, int Dkept, int Gtot, int T, int A, const double* rec_thrs, int R,
                         const int* max_dets, int M, void* workspace, size_t workspace_bytes, double* precision,
                         double* recall, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Image-space masks and COCO RLE (csrc/mask_rle.cu): detectron2's GPU paste_masks_in_image + threshold, pycocotools
 * rleEncode + rleToString, and the decode + confusion counts of the reference's mask tools.  mode picks how a map
 * becomes probabilities: 0 as given, 1 = L1 ((p - min) / (max - min) per map), 2 = sigmoid.  threshold must be > 0.
 *
 * gdrn_mask_paste: masks [n,mh,mw] f32, boxes [n,4] f32 XYXY -> out [n,H,W] u8 (0 / 1).
 * gdrn_mask_paste_rle: maps0 (and maps1, or null) [n,1,mh,mw] f32, the box of ROI i is roi_center[i] -/+ scale[i] / 2
 *   (f32).  S = n (2n with maps1) strings, string s = kind * n + roi, packed in string order into chars (at least
 *   S * gdrn_mask_rle_max_chars(H, W) bytes); table [S,2] i64 = (offset, length).  workspace:
 *   gdrn_mask_rle_workspace_bytes(S, H, W) bytes.  No synchronisation.
 * gdrn_rle_confusion: P compressed strings (chars + table [P,2] (offset, length)) decoded at H x W against gt [P,H,W] u8
 *   (row-major, nonzero = set) -> counts [P,4] i64 = TP, FP, FN, TN; status [P] i32 device scratch.  Synchronises the
 *   stream; a malformed string (bad char, unterminated group, total != H * W) is an error naming the string.
 * ------------------------------------------------------------------------------------------- */
int gdrn_mask_paste(const float* masks, int n, int mh, int mw, int mode, const float* boxes, int H, int W, float threshold,
                    uint8_t* out, void* stream);
size_t gdrn_mask_rle_max_chars(int H, int W);
size_t gdrn_mask_rle_workspace_bytes(int S, int H, int W);
int gdrn_mask_paste_rle(const float* maps0, const float* maps1, int n, int mh, int mw, int mode, const float* roi_center,
                        const float* scale, int H, int W, float threshold, void* workspace, size_t workspace_bytes,
                        char* chars, size_t chars_bytes, long long* table, void* stream);
int gdrn_rle_confusion(const char* chars, size_t chars_bytes, const long long* table, int P, const uint8_t* gt, int H, int W,
                       int* status, long long* counts, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Ground-truth annotations of a BOP split (csrc/gt_info.cu): the per-instance math of calc_gt_info.py and
 * calc_gt_masks.py for n instances of N images of one size H x W.  Results do not depend on the launch shape.
 *
 * gdrn_gt_info: depth_large [n,3H,3W] f32 is instance i rendered alone (float z, 0 = background) on the 3x canvas with
 *   principal point (cx + W, cy + H); depth_img [n,H,W] f32 (or null) the same instance at image size with K.
 *   depth_test [N,H,W] u16 sensor depth, depth_scale [N] f32, Ks [N,3,3] f64; instance i lies in image inst_img[i]
 *   (i32).  The test depth is f32(u16) * depth_scale in f32; distances and bop19 visibility (diff in f32 against delta)
 *   are the ones VSD uses.  counts [n,3] i64 = px_count_all (canvas coverage), px_count_valid, px_count_visib;
 *   boxes [n,8] i32 = bbox_obj, bbox_visib as (x_min, y_min, x_max - x_min, y_max - y_min), bbox_obj in image
 *   coordinates (may be negative or extend past the image), both -1 unless px_count_visib > 0.  With depth_img,
 *   mask / mask_visib [n,H,W] u8 = 0 / 255.  depth_large may be null when depth_img is given (masks only: counts 0,
 *   boxes -1).  Allocates nothing, does not synchronise.
 * ------------------------------------------------------------------------------------------- */
int gdrn_gt_info(const float* depth_large, const float* depth_img, const uint16_t* depth_test, const float* depth_scale,
                 const double* Ks, const int* inst_img, int n, int H, int W, float delta, long long* counts, int* boxes,
                 uint8_t* mask, uint8_t* mask_visib, void* stream);

/* ---------------------------------------------------------------------------------------------
 * xyz_crop training targets of a BOP split (csrc/xyz_crop.cu): the per-instance math of the *_1_gen_xyz.py scripts for
 * n instances rendered alone at one size H x W (depth [n,H,W] f32, float z, 0 = background).
 *   gdrn_xyz_crop_boxes: boxes [n,4] i32 = x1, y1, x2, y2, the inclusive pixel box of depth != 0; an empty render gives
 *     (INT_MAX, INT_MAX, INT_MIN, INT_MIN).  Integer min / max only: independent of the launch shape.
 *   gdrn_xyz_crop_pack: R [n,9] (row-major cam_R_m2c), t [n,3] (metres), K [n,9], all f32; boxes from
 *     gdrn_xyz_crop_boxes; offsets [n] i64 in fp16 elements.  Writes instance i's crop at out + offsets[i] as
 *     [y2-y1+1, x2-x1+1, 3] fp16 (round to nearest even) of R^T (((u - cx) z / fx, (v - cy) z / fy, z) - t), computed
 *     in f32 with the product rounded before the division, and 0 where z == 0; an empty instance gets [H, W, 3] zeros.
 * Allocate nothing, do not synchronise.
 * ------------------------------------------------------------------------------------------- */
int gdrn_xyz_crop_boxes(const float* depth, int n, int H, int W, int* boxes, void* stream);
int gdrn_xyz_crop_pack(const float* depth, const float* R, const float* t, const float* K, const int* boxes,
                       const long long* offsets, int n, int H, int W, uint16_t* out, void* stream);


/* ---------------------------------------------------------------------------------------------
 * Pose visualisation composite (csrc/vis_poses.cu): the pixel arithmetic of visualization.vis_object_poses
 * (lib/pysixd/visualization.py) for N images of one size H x W; image j owns instances [inst_off[j], inst_off[j+1])
 * of the n instance renders, in drawing order; max_inst >= the largest inst_off[j+1] - inst_off[j] (at most 3000).
 *   m_rgb [n,H,W,3] u8 and m_depth [n,H,W] f32 (rast_render_meshes_rgb), rgb [N,H,W,3] u8, depth [N,H,W] f32 in mm.
 *   flags: 1 = rgb visualisation, 2 = resolve visibility, 4 = depth difference.
 *   -> ren_rgb [N,H,W,3] u8 (resolved, or the saturating sum), ren_depth [N,H,W] f32, blend [N,H,W,3] u8 =
 *      floor(0.5 * rgb + 0.5 * ren_rgb), boxes [n,4] i32 = x_min, y_min, x_max, y_max of m_rgb > 0 (INT_MAX,
 *      INT_MAX, INT_MIN, INT_MIN when empty); diff_vis [N,H,W,3] u8 (the depth-difference image without text),
 *      diff_minmax [N,2] f32, diff_sum [N] f64, diff_count [N] i64 over the valid pixels.  Every output is
 *      independent of the order in which CTAs run.  workspace of gdrn_vis_poses_workspace_bytes(N, H, W) bytes.
 * ------------------------------------------------------------------------------------------- */
size_t gdrn_vis_poses_workspace_bytes(int N, int H, int W);
int gdrn_vis_poses(const uint8_t* m_rgb, const float* m_depth, const int* inst_off, int max_inst, int N, int n,
                   const uint8_t* rgb,
                   const float* depth, int H, int W, int flags, uint8_t* ren_rgb, float* ren_depth, uint8_t* blend,
                   int* boxes, uint8_t* diff_vis, float* diff_minmax, double* diff_sum, long long* diff_count,
                   void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training batch pipeline (csrc/train_aug.cu): read_data_train's image work for n uint8 BGR images [n,H,W,3] of one size.
 *   gdrn_train_composite: mask_visib [n,H,W] u8 (0/1); bbox [n,4] i32 the host sets to (H, -1, W, -1) -> the visible
 *     mask's row / column extent; side [n] (0 top, 1 bottom, 2 left, 3 right, else none) and trunc_u [n] in [0, 1) ->
 *     keep [n,4] = row0, row1, col0, col1 of the truncated mask; bg_meta [n,7] = do_bg, bg_h, bg_w, crop_h, crop_w,
 *     resized_h, resized_w; bg_scale [n,2] = 1 / fx, 1 / fy; background j at bg_pool + bg_off[j] (u8 [bg_h,bg_w,3]).
 *     Pixels outside the kept mask of a do_bg image become the resized background (0 beyond it), in place.
 *   gdrn_train_luma_sum: sums [n] u64 = sum of PIL's L image of each image whose kind_at[b][step] is EnhanceContrast.
 *   gdrn_train_color_step: dst = colour op kind_at[b][step] (kinds 0..11, others pass through) of src with params
 *     fpar [n,S,4] f32, ipar [n,S,12] i32, dropout cells [n,ch,cw] u8, luma_sums from gdrn_train_luma_sum.
 *   gdrn_train_roi_crop: center_scale [n,3] f64 -> roi_img [n,3,in,in] (normalised), roi_coord_2d [n,2,out,out],
 *     roi_mask_trunc / visib / full [n,out,out] f32 (nearest), counts [n,2] i32 = trunc and visib pixels of each ROI.
 * Allocate nothing, do not synchronise.
 * ------------------------------------------------------------------------------------------- */
int gdrn_train_composite(uint8_t* images, const uint8_t* mask_visib, int n, int H, int W, const uint8_t* bg_pool,
                         const long long* bg_off, const int* bg_meta, const double* bg_scale, const int* side,
                         const double* trunc_u, int* bbox, int* keep, void* stream);
int gdrn_train_luma_sum(const uint8_t* images, int n, int H, int W, const int* kind_at, int S, int step,
                        unsigned long long* sums, void* stream);
int gdrn_train_color_step(const uint8_t* src, uint8_t* dst, int n, int H, int W, const int* kind_at, const float* fpar,
                          const int* ipar, int S, int step, const uint8_t* cells, int ch, int cw,
                          const unsigned long long* luma_sums, void* stream);
int gdrn_train_roi_crop(const uint8_t* images, const uint8_t* mask_visib, const uint8_t* mask_full, const int* keep,
                        const double* center_scale, int n, int H, int W, int in_res, int out_res, const double* pixel_mean,
                        const double* pixel_std, float* roi_img, float* roi_coord_2d, float* roi_mask_trunc,
                        float* roi_mask_visib, float* roi_mask_full, int* counts, void* stream);

/* ---------------------------------------------------------------------------------------------
 * YOLOX training batch pipeline (csrc/yolox_train_aug.cu): MosaicDetection + TrainTransform's image work on uint8 BGR
 * images (HWC, 3 channels), oh x ow the training size.  Offsets are in bytes from the named pool's base.
 *   yolox_train_resize: jobs [n_jobs,8] i64 = src_off, sh, sw, dst_off, dh, dw, ch, cw: dst (ch x cw) = the source resized
 *     to dh x dw (cv2.resize INTER_LINEAR) top-left, 114 elsewhere; max_plane >= every ch * cw.
 *   yolox_train_mosaic_affine: tile_info [n_sel,4,8] i64 = lx1, ly1, lx2, ly2, padw, padh, tile_w, tile_off (tiles pasted
 *     in order into a 2oh x 2ow mosaic of 114), M [n_sel,6] f64 the forward affine -> out[sel[i]] = cv2.warpAffine of the
 *     mosaic to (ow, oh), bilinear, border 114.
 *   yolox_train_mixup: params [n_sel,6] i64 = canvas_off, jit_h, jit_w, flip, x_offset, y_offset; canvas (oh x ow) resized
 *     to jit_h x jit_w, mirrored when flip, zero-padded and cropped at the offsets, blended 0.5 / 0.5 into images[sel[i]].
 *   yolox_train_hsv: entries [n,2] i64 = off, npix; luts [n,3,256] u8 (hue, saturation, value); rgb: channel 0 is R.
 *     In place; max_pix >= every npix.
 *   yolox_train_preproc: info [n,5] i64 = src_off, sh, sw, flip, transpose -> out [n,oh,ow,3] = the mirrored source
 *     letterboxed into 114 (TrainTransform's preproc), stored as (ow, oh, 3) when transpose.
 *   yolox_train_pack: images [n,oh,ow,3] (transposed[b]: stored (ow, oh, 3)) -> out [n,3,oh,ow] f32.
 * Allocate nothing, do not synchronise.
 * ------------------------------------------------------------------------------------------- */
int yolox_train_resize(const uint8_t* src, uint8_t* dst, const long long* jobs, int n_jobs, long long max_plane, void* stream);
int yolox_train_mosaic_affine(const uint8_t* tiles, const long long* tile_info, const double* M, const int* sel, int n_sel,
                              int oh, int ow, uint8_t* out, void* stream);
int yolox_train_mixup(uint8_t* images, const uint8_t* canvases, const long long* params, const int* sel, int n_sel, int oh,
                      int ow, void* stream);
int yolox_train_hsv(uint8_t* pool, const long long* entries, const uint8_t* luts, int n, long long max_pix, int rgb,
                    void* stream);
int yolox_train_preproc(const uint8_t* pool, const long long* info, int n, int oh, int ow, uint8_t* out, void* stream);
int yolox_train_pack(const uint8_t* images, const int* transposed, int n, int oh, int ow, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Parameter update of both trainers (csrc/train_step.cu): one step of Ranger (lib/torch_utils/solver/ranger.py: GC,
 * RAdam, lookahead) over every parameter of a model in one launch, and the model EMA (det/yolox/utils/ema.py,
 * lib/torch_utils/torch_utils.py ModelEMA) in one launch.  DESIGN.md §7s pins every rule.
 *
 * GdrnRangerParam: one fp32 parameter with a gradient, dense with dim 0 outermost; grad, exp_avg, exp_avg_sq and
 *   slow_buffer have the parameter's strides.  The caller fills param .. row_len, flags and the scalars;
 *   gdrn_ranger_plan fills unit_begin, mean_begin, units, rows_per_unit and path on the host.
 *   row_len = numel / size(0) (the GC mean length).  flags: 1 gradient centralisation (grad is replaced in place by
 *   grad - mean over each dim-0 slice), 2 state created this step (moments read as 0, slow_buffer = the parameter
 *   before the update), 4 weight decay (p += neg_wd_lr * p first), 8 adaptive branch (p += neg_step_lr * exp_avg /
 *   (sqrt(exp_avg_sq) + eps); else p += neg_step_lr * exp_avg), 16 lookahead (slow += alpha (p - slow); p = slow).
 * gdrn_ranger_plan: host only.  n_units = the update grid; n_long_rows = the dim-0 slices longer than the on-chip bound
 *   (their means come from a separate fixed-order pass into the workspace).
 * gdrn_ranger_workspace_bytes(n_long_rows): workspace of gdrn_ranger_step.
 * gdrn_ranger_step: params = the planned table in DEVICE memory.  One launch, two with long rows.  Results do not
 *   depend on the launch order of CTAs.
 * GdrnEmaEntry / gdrn_ema_plan / gdrn_ema_update: ema = fl(fl(ema * decay) + fl(one_minus_decay * model)) per element,
 *   no FMA, over every entry of the DEVICE table (ema and model of equal numel and strides, dense); one launch.
 * ------------------------------------------------------------------------------------------- */
typedef struct GdrnRangerParam {
  float* param;
  float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  float* slow_buffer;
  long long numel;
  long long row_len;
  long long unit_begin;
  long long mean_begin;
  int units;
  int flags;
  float beta1, one_minus_beta1, beta2, one_minus_beta2;
  float neg_step_lr, neg_wd_lr, eps, alpha;
  int rows_per_unit;
  int path;
  long long reserved;
} GdrnRangerParam; /* 128 bytes */

typedef struct GdrnEmaEntry {
  float* ema;
  const float* model;
  long long numel;
  long long unit_begin;
} GdrnEmaEntry; /* 32 bytes */

int gdrn_ranger_plan(GdrnRangerParam* params, int n, long long* n_units, long long* n_long_rows);
size_t gdrn_ranger_workspace_bytes(long long n_long_rows);
int gdrn_ranger_step(const GdrnRangerParam* params, int n, long long n_units, long long n_long_rows, void* workspace,
                     size_t workspace_bytes, void* stream);
int gdrn_ema_plan(GdrnEmaEntry* entries, int n, long long* n_units);
int gdrn_ema_update(const GdrnEmaEntry* entries, int n, long long n_units, float decay, float one_minus_decay,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GDRN_B200_H_ */
