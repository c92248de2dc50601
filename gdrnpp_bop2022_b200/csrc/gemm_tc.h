// Internal C++ interface of the wgmma/TMA implicit-GEMM kernel (gemm_tc.cu).
//
//   D[m, n] = sum_{tap} sum_{k} A_tap[m, k] * W[n, tap.b_off + k]      (bf16 x bf16 -> fp32)
//
// A rows are pixels of an NHWC activation tensor: a 128-row tile is a (bw x bh x bb) box of pixels
// fetched by one TMA box load per (tap, k-chunk); conv padding = TMA out-of-bounds zero fill.  The k-chunk width (32
// for split-bf16 convolutions, 64 otherwise) is chosen by gemm_tc_launch, which encodes both operand maps from the plan's
// a_* / b_* geometry.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

enum GemmEpilogue : int {
  EPI_STORE = 0,      // out = acc (+bias)                      -> bf16 or fp32
  EPI_GELU = 1,       // out = gelu(acc + bias)                 -> bf16
  EPI_RESID = 2,      // out = resid + gamma * (acc + bias)     -> fp32 (in place allowed)
  EPI_GNSTATS = 3,    // out = acc; per-(image, group) sum / sumsq accumulated in double
  EPI_BIAS_LN = 4,    // out = LayerNorm_C(acc + bias) * ln_w + ln_b  (N == BLOCK_N)  -> fp32
  EPI_OUTCONV = 5,    // class-gathered geometry-head output + Patch-PnP input assembly
};

struct GemmTap {
  int c0;     // added to coordinate 0 (channel offset; e.g. x-parity * C for the stride-2 view, or the lo-half offset)
  int d1;     // added to coordinate 1 (x; rank 2: row offset)
  int d2;     // rank 4: added to y.  rank 5: absolute coordinate 2 (y parity)
  int d3;     // rank 5: added to y (coordinate 3)
  int b_off;  // K offset of this tap inside a row of W (elements)
};

constexpr int GEMM_MAX_TAPS = 27;  // 9 spatial taps x 3 split-bf16 products

struct GemmPlan {
  // ---- A operand ----
  CUtensorMap tmap_a;   // set by gemm_tc_launch from a_ptr / a_dims / a_str / a_box
  int a_rank;           // 2: plain [M,K] rows; 4: (C,W,H,B); 5: (2C, W/2, 2, H/2, B) stride-2 view
  const void* a_ptr;    // A base
  uint64_t a_dims[5];   // tensor dims, innermost (channels) first
  uint64_t a_str[4];    // byte strides of dims 1..a_rank-1
  uint32_t a_box[5];    // pixel box of dims 1..a_rank-1 (a_box[0], the k-chunk width, is set by gemm_tc_launch)
  int a_k;              // K per tap (elements)
  int lg_bw, lg_bh, lg_bb;  // log2 of the pixel box (bw*bh*bb == 128); rank 2 ignores them
  int tiles_x, tiles_y;     // tiles per image along x / y (rank 4/5)
  int num_taps;
  GemmTap taps[GEMM_MAX_TAPS];
  int k_chunks;         // set by gemm_tc_launch: ceil(a_k / k-chunk width)
  // ---- B operand ----
  CUtensorMap tmap_b;   // 2D [rows][K_total] bf16, K-major; set by gemm_tc_launch from b_ptr / b_rows / b_ktot
  int b_rows_per_class; // EPI_OUTCONV: row offset multiplier for the ROI class (0 otherwise)
  const void* b_ptr;    // W base / rows / row length (elements)
  long long b_rows, b_ktot;
  // ---- problem ----
  int m_tiles, n_tiles;  // tile t is (m_tile, n_tile) = (t / n_tiles, t % n_tiles): consecutive CTAs share an A tile
  int M;                // valid rows (rank 2) ; rank 4/5: number of images B
  int N;                // valid output columns
  // ---- epilogue ----
  int epi;
  int out_f32;          // EPI_STORE / EPI_GNSTATS: 1 -> fp32 output, 0 -> bf16
  int gelu_mode;        // EPI_GELU: 0 = fp32 ex2/rcp form (1.2e-5 of erf), 1 = packed half2 tanh.approx, 2 = fp32 tanh.approx, 3 = erff
                        // (bf16 plans; a split GELU is always the erf form, mode 3, whatever this field says)
  int split;            // split-bf16 (x3) mode: operands are [hi | lo] pairs (see x3_*), bf16 outputs are written as
                        // [hi | lo] pairs (row width 2N, lo = bf16(v - hi))
  int x3_a_lo;          // split: offset of the lo half in A's coordinate 0 (channels / K); taps[] list the hi operands only
  int x3_b_lo;          // split: offset of the lo half inside a row of W (elements)
  void* out;            // [rows, ldo]
  CUtensorMap tmap_out; // rank-2 outputs: store map (filled by gemm_tc_launch when use_tma_store)
  int use_tma_store;    // set by gemm_tc_launch
  int resid_reduce;     // set by gemm_tc_launch: EPI_RESID in place -> TMA reduce-add (x += gamma*(acc+bias)), x is never read by the SM
  long long ldo;        // output row stride (elements)
  int OH, OW, osy, osx, ooy, oox;  // rank 4/5: out row = (b*OH + y*osy+ooy)*OW + x*osx+oox
  const float* bias;    // [N] or null
  const float* gamma;   // EPI_RESID [N]
  const float* resid;   // EPI_RESID [rows, ldo] fp32
  double* gn_stats;     // EPI_GNSTATS [B, groups, 2]
  int gn_groups, gn_cpg;    // groups per image, channels per group
  const float* ln_w; const float* ln_b; float ln_eps;  // EPI_BIAS_LN
  int ln_n;             // EPI_BIAS_LN: LayerNorm width (0 = N); columns [ln_n, N) are zero PAD channels (zero weight rows / bias / affine)
  // EPI_OUTCONV
  const long long* roi_classes;  // [B]; NULL = class 0 for every ROI (class-agnostic head)
  int num_classes;               // roi_classes are clamped to [0, num_classes)
  int rows_per_roi;              // 4096
  const float* oc_bias;          // [num_classes, 80]
  const float* roi_extents;      // [B,3]
  const float* roi_coord_2d;     // [B,2,64,64] fp32 NCHW
  void* pnp_in;                  // bf16 [B*4096, 128]
  float* map_mask; float* map_full; float* map_x; float* map_y; float* map_z; float* map_region;  // NCHW or null
};

// block_n in {16, 64, 80, 128, 256} (256: run as 128-wide tiles)
int gemm_tc_launch(const GemmPlan& plan, int block_n, cudaStream_t stream);

// Ids of the launch record (gdrn_gemm_kernels_launched): gemm_tc_launch's instantiations take 0 .. GEMM_NUM_TC_KERNELS - 1
// in the order of gemm_tc.cu's kGemmKernels table, the fused MLP kernels the two after them.
constexpr int GEMM_NUM_TC_KERNELS = 20;
constexpr int GEMM_KERNEL_ID_MLP_FUSED = GEMM_NUM_TC_KERNELS;
constexpr int GEMM_KERNEL_ID_MLP_FUSED_X3 = GEMM_NUM_TC_KERNELS + 1;
static_assert(GEMM_KERNEL_ID_MLP_FUSED_X3 < 64, "gemm: the launch record is one 64-bit mask");

// Fused ConvNeXt MLP block (C = 128, mlp_fused.cu): x += gamma * (W2 . gelu(W1 . A + b1) + b2), hidden activation kept on
// chip.  A bf16 [M, C]; W1 bf16 [4C, C]; W2 bf16 [C, 4C]; x fp32 [M, C] updated in place.
// split-bf16 (parity mode) twin: A [M,2C], W1 [4C,2C], W2 [C,8C] hold [hi | lo] halves
int mlp_fused_x3_supported(int C, long long M);
int mlp_fused_x3_launch(const void* A, const void* W1, const float* b1, const void* W2, const float* b2, const float* gamma,
                        float* x, long long M, int C, cudaStream_t stream);
int mlp_fused_supported(int C, long long M);
int mlp_fused_launch(const void* A, const void* W1, const float* b1, const void* W2, const float* b2, const float* gamma,
                     float* x, long long M, int C, cudaStream_t stream);

// tensor-map builders (bf16). dims/strides innermost first; strides in BYTES for dims 1..rank-1.
// fp32, no swizzle, zero OOB fill (dense [..][box0] shared-memory image)
int make_tmap_f32_plain(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box);
int make_tmap_store(CUtensorMap* out, const void* base, int is_f32, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box);
// same for narrow tiles: 64-byte rows use SWIZZLE_64B (16-byte chunk c of row r at c ^ ((r >> 1) & 3): conflict-free
// row-wise STS.128), anything else SWIZZLE_NONE (dense [rows][box0] shared-memory tile)
int make_tmap_store_plain(CUtensorMap* out, const void* base, int is_f32, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box);
// K-major operand tiles: box[0] of 64 elements (128-byte rows) uses SWIZZLE_128B, of 32 elements (64-byte rows) SWIZZLE_64B
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);
