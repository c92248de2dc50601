// Depthwise 7x7 + bias + LayerNorm(C) -> GEMM A operand: PERSISTENT, two-warpgroup ping-pong version for the
// 16x8-pixel x 64-channel tiles of ConvNeXt stages 0-2 (33 of the 36 blocks).  Reference op: timm ConvNeXtBlock
// conv_dw (7x7, groups = C) -> LayerNorm(C, eps 1e-6) (third-party timm 0.6.7, un-vendored).
//
// Why: the one-tile-per-CTA kernel (dense_ops.cu, dwconv_ln_cluster_kernel) spends only ~40 % of a CTA's life in the
// convolution (FMA pipe); TMA load wait, the LayerNorm exchange across the channel-slice cluster and the output stores do
// not overlap it, and the two CTAs resident on an SM run those phases in lock-step (profiles/r01_dwconv_experiments.md:
// 41 % FMA-pipe active, 0.99 TB/s).  Here one CTA per SM stays resident and loops over pixel tiles with TWO warpgroups
// (2 x 8 warps) in ping-pong, each with its own shared-memory halo slot:
//     WG0:  conv(t0) | LN/exchange/store(t0) + TMA(t2) | conv(t2) | ...
//     WG1:           | conv(t1)                        | LN/exchange/store(t1) + TMA(t3) | conv(t3) ...
// A pair of named barriers hands the FMA pipe from one warpgroup to the other, so the convolutions never overlap each
// other but everything else (load wait, LN shuffles, DSMEM pushes, stores) runs underneath the other warpgroup's
// convolution.  The 49 x 64 filter taps of the CTA's channel slice are loaded once per launch.
//
// Cluster = the C/64 CTAs holding the channel slices of the same pixel-tile sequence (as before): per tile every warp
// pushes its 64-channel (sum, M2) partials into all peers with st.async + mbarrier complete_tx (data and signal travel
// together), double-buffered per warpgroup so that a fast peer can never overwrite partials that are still being read.
#include <cooperative_groups.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "dense_ops.h"
#include "dw_helpers.cuh"
#include "gemm_tc.h"

namespace cg = cooperative_groups;

namespace {

__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

constexpr int PP_TW = 16, PP_TH = 8, PP_CPC = 64;
constexpr int PP_IW = PP_TW + 6, PP_IH = PP_TH + 6;
constexpr int PP_NPIX = PP_TW * PP_TH;                      // 128
constexpr int PP_WG_THREADS = (PP_CPC / 2) * PP_TH;         // 256: lane = channel pair, warp = output row
constexpr int PP_SLOT_FLOATS = PP_IH * PP_IW * PP_CPC;      // 19 712 floats = 78 848 B
constexpr int PP_MAX_RANKS = 8;
constexpr size_t PP_SMEM = (size_t)(2 * PP_SLOT_FLOATS + 49 * PP_CPC) * 4 + (size_t)2 * 2 * PP_MAX_RANKS * PP_NPIX * 8 + 64 +
                           (size_t)2 * PP_NPIX * 8 + 64;   // halo slots, taps, partials, barriers, (mean, rstd) per warpgroup

// NR = channel slices (cluster size, C = 64 * NR), SPLIT = [hi C | lo C] bf16 output rows, TRACE = phase cycle counters.
// Everything that depends on (C, split) is a compile-time constant: the kernel is instruction-issue bound (the code around
// the convolution was ~1.2 k dynamic instructions per thread and tile against 0.98 k for the convolution itself), so output
// strides are immediates, the Chan combine is unrolled, and the normalisation runs in packed fp32.
// R2 = the convolution's thread tile: false = one output row x 16 pixels per thread (warp = output row: 22 halo + 7 tap
// LDS.64 per filter row, 203 per tile), true = TWO output rows x 8 pixels (warp = row pair x half of the tile width): an
// input row is loaded once for both output rows and a filter row's taps are kept for the second one, 161 LDS.64 per tile for
// the same 784 FMA pairs, same per-output accumulation order (bit-identical results).
template <int NR, bool SPLIT, bool TRACE, bool R2 = false>
__global__ void __launch_bounds__(2 * PP_WG_THREADS, 1)
dwconv_ln_pp_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                    const float* __restrict__ bias, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                    __nv_bfloat16* __restrict__ out, int B, int H, int W, int c_real, float eps, int use_token,
                    long long* trace) {
  constexpr int TW = PP_TW, TH = PP_TH, CPC = PP_CPC, IW = PP_IW, NPIX = PP_NPIX;
  constexpr int C = NR * CPC;
  constexpr int LDC = SPLIT ? 2 * C : C;
  // experiment bits (GDRN_DW_DBG, wrong results): 8 = no output stores, 16 = no cluster exchange (own partial only), 32 = no convolution
  const int dbg = use_token >> 3;
  use_token &= 1;
  constexpr int NV = TW;              // pixels per thread (one output row)
  constexpr int LPP = 32 / NV;        // lanes per pixel after the transposing reduction (2)
  extern __shared__ __align__(1024) float smem_pp[];
  float* slot0 = smem_pp;                                        // [2][IH][IW][CPC] halo tiles (TMA destinations)
  float* wsm = smem_pp + 2 * PP_SLOT_FLOATS;                     // [49][CPC]
  float2* parts = reinterpret_cast<float2*>(wsm + 49 * CPC);     // [2 wg][2 buf][MAX_RANKS][NPIX]
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(parts + 2 * 2 * PP_MAX_RANKS * NPIX);
  float2* stats = reinterpret_cast<float2*>(bars + 8);           // [2 wg][NPIX] (mean, rstd) of the tile being normalised
  // bars: [0] weights, [1..2] tile loaded (per wg), [3..6] partials (wg * 2 + buf)

  ptx::griddep_launch();
  const int rank = (int)ptx::cluster_ctarank();
  const int cluster_id = blockIdx.x / NR, nclusters = gridDim.x / NR;
  const int c0 = rank * CPC;
  const int tiles_x = W / TW, tiles_y = H / TH;
  const int n_tiles = B * tiles_x * tiles_y;
  const int n_my = cluster_id < n_tiles ? (n_tiles - cluster_id + nclusters - 1) / nclusters : 0;
  const int wg = threadIdx.x >> 8;
  const int tidw = threadIdx.x & 255, lane = tidw & 31;
  const int row0 = tidw >> 5;          // output row of this warp
  const int rp2 = (row0 >> 1) * 2, xh8 = (row0 & 1) * 8;   // R2: first output row / first output column of this warp
  const int cl = 2 * lane;             // first channel of the pair (CTA-local)
  const int n_w = (n_my - wg + 1) >> 1;                    // tiles of this warpgroup: k = wg, wg + 2, ...
  const int n_other = (n_my - (wg ^ 1) + 1) >> 1;
  float* tile = slot0 + wg * PP_SLOT_FLOATS;

  const uint32_t bar_w = ptx::smem_u32(bars);
  const uint32_t bar_tile = ptx::smem_u32(bars + 1 + wg);
  auto bar_parts = [&](int buf) { return ptx::smem_u32(bars + 3 + wg * 2 + buf); };
  constexpr uint32_t parts_bytes = (uint32_t)(NR * NPIX * sizeof(float2));
  if (threadIdx.x == 0) {
    for (int i = 0; i < 7; ++i) ptx::mbar_init(ptx::smem_u32(bars + i), 1);
    ptx::fence_barrier_init();
    // every (rank, pixel) partial of the cluster lands as one 8-byte st.async on the barrier of its (wg, buffer)
    for (int i = 3; i < 7; ++i) ptx::mbar_arrive_expect_tx(ptx::smem_u32(bars + i), parts_bytes);
  }
  __syncthreads();
  // tile sequence of this warpgroup: t = cluster_id + (wg + 2 i) * nclusters; (x, y, b) advance incrementally (no divisions per tile)
  const int tiles_img = tiles_x * tiles_y;
  int t_cur = cluster_id + wg * nclusters;
  int tb = t_cur / tiles_img, trem = t_cur - tb * tiles_img;
  const int step = 2 * nclusters;
  const int step_b = step / tiles_img, step_r = step - step_b * tiles_img;
  auto coords = [&](int b_, int rem_, int& b, int& y0, int& x0) {
    const int ty = rem_ / tiles_x;     // tiles_x is 1, 2 or 4 here: the compiler cannot know, one division per tile and thread
    b = b_; y0 = ty * TH; x0 = (rem_ - ty * tiles_x) * TW;
  };
  if (threadIdx.x == 0) {
    ptx::mbar_arrive_expect_tx(bar_w, (uint32_t)(49 * CPC * sizeof(float)));
    ptx::tma_load_2d(ptx::smem_u32(wsm), &tmap_w, bar_w, c0, 0);          // this CTA's 49 x 64 filter taps, once
  }
  ptx::griddep_wait();   // barriers and the (constant) filter taps were set up under the previous kernel's tail
  if (tidw == 0 && n_w > 0) {
    int b, y0, x0;
    coords(tb, trem, b, y0, x0);
    ptx::mbar_arrive_expect_tx(bar_tile, (uint32_t)(PP_SLOT_FLOATS * sizeof(float)));
    ptx::tma_load_4d(ptx::smem_u32(tile), &tmap_x, bar_tile, c0, x0 - 3, y0 - 3, b);
  }
  ptx::cluster_sync_all();     // every peer's barriers exist and are armed before the first push (once per launch)
  const f32x2_t bv = f2_pack(__ldg(bias + c0 + cl), __ldg(bias + c0 + cl + 1));
  const f32x2_t gw = f2_pack(__ldg(ln_w + c0 + cl), __ldg(ln_w + c0 + cl + 1));
  const f32x2_t gb = f2_pack(__ldg(ln_b + c0 + cl), __ldg(ln_b + c0 + cl + 1));
  ptx::mbar_wait(bar_w, 0);

  // GDRN_DW_TRACE: phase cycle counts of warpgroup 0 / thread 0 of one mid-grid CTA, summed over its tiles
  const bool trc = TRACE && trace != nullptr && blockIdx.x == (gridDim.x / 2) && threadIdx.x == 0;
  long long tt[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  long long tq = trc ? clock64() : 0;
#define PP_MARK(slot) do { if constexpr (TRACE) { if (trc) { const long long t_ = clock64(); tt[slot] += t_ - tq; tq = t_; } } } while (0)
  for (int i = 0; i < n_w; ++i) {
    int b, y0, x0;
    coords(tb, trem, b, y0, x0);
    // next tile of this warpgroup
    trem += step_r; tb += step_b;
    if (trem >= tiles_img) { trem -= tiles_img; ++tb; }
    ptx::mbar_wait(bar_tile, (uint32_t)(i & 1));          // halo tile landed
    PP_MARK(0);
    // ---- FMA-pipe hand-over: the convolutions of the two warpgroups alternate ----
    if (use_token) {
      if (wg == 0) { if (i > 0) named_bar_sync(2, 2 * PP_WG_THREADS); }
      else named_bar_sync(1, 2 * PP_WG_THREADS);
    }
    PP_MARK(1);
    f32x2_t acc[TW];
#pragma unroll
    for (int ox = 0; ox < TW; ++ox) acc[ox] = bv;
    if constexpr (R2) {
      // acc[r * 8 + q] = output (rp2 + r, xh8 + q).  Input row iy feeds output row 0 with filter row iy and output row 1 with
      // filter row iy - 1 (the taps loaded one iteration earlier): per output the order is still ky = 0..6, kx = 0..6.
      f32x2_t wprev[7];
#pragma unroll
      for (int iy = 0; iy < 8; ++iy) {
        f32x2_t v[14], wk[7];
        const float* rowp = tile + ((rp2 + iy) * IW + xh8) * CPC + cl;
#pragma unroll
        for (int j = 0; j < 14; ++j) v[j] = *reinterpret_cast<const f32x2_t*>(rowp + j * CPC);
        if (iy < 7) {
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) wk[kx] = *reinterpret_cast<const f32x2_t*>(wsm + (iy * 7 + kx) * CPC + cl);
#pragma unroll
          for (int kx = 0; kx < 7; ++kx)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = f2_fma(v[q + kx], wk[kx], acc[q]);
        }
        if (iy >= 1) {
#pragma unroll
          for (int kx = 0; kx < 7; ++kx)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[8 + q] = f2_fma(v[q + kx], wprev[kx], acc[8 + q]);
        }
        if (iy < 7) {
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) wprev[kx] = wk[kx];
        }
      }
    } else if (!(dbg & 4)) {
#pragma unroll
    for (int ky = 0; ky < 7; ++ky) {
      f32x2_t v[IW], wk[7];
      const float* rowp = tile + ((row0 + ky) * IW) * CPC + cl;
#pragma unroll
      for (int j = 0; j < IW; ++j) v[j] = *reinterpret_cast<const f32x2_t*>(rowp + j * CPC);
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) wk[kx] = *reinterpret_cast<const f32x2_t*>(wsm + (ky * 7 + kx) * CPC + cl);
#pragma unroll
      for (int kx = 0; kx < 7; ++kx)
#pragma unroll
        for (int ox = 0; ox < TW; ++ox) acc[ox] = f2_fma(v[ox + kx], wk[kx], acc[ox]);
    }
    }
    PP_MARK(2);
    if (use_token) {
      if (wg == 0) { if (i < n_other) named_bar_arrive(1, 2 * PP_WG_THREADS); }
      else { if (i + 1 < n_other) named_bar_arrive(2, 2 * PP_WG_THREADS); }
    }
    // the whole warpgroup has finished reading its halo slot: prefetch the next tile into it
    named_bar_sync(3 + wg, PP_WG_THREADS);
    if (tidw == 0 && i + 1 < n_w) {
      int nb, ny0, nx0;
      coords(tb, trem, nb, ny0, nx0);
      ptx::mbar_arrive_expect_tx(bar_tile, (uint32_t)(PP_SLOT_FLOATS * sizeof(float)));
      ptx::tma_load_4d(ptx::smem_u32(tile), &tmap_x, bar_tile, c0, nx0 - 3, ny0 - 3, nb);
    }
    PP_MARK(3);
    // ---- LayerNorm statistics of this warp's 64 channels (shuffles only) ----
    // Zero pad channels (c >= c_real, all in the last slice) are left out of the slice's mean and M2.
    // pixel (tile-local index) of value q of this thread: R2 maps q -> (row rp2 + q / 8, column xh8 + q % 8)
    const int vi = lane / LPP;
    const int pix = R2 ? (rp2 + (vi >> 3)) * TW + xh8 + (vi & 7) : row0 * TW + vi;
    float s_loc, m2_loc;
    {
      const float inv_n = 1.0f / (float)min(CPC, c_real - c0);
      const bool real_x = c0 + cl < c_real, real_y = c0 + cl + 1 < c_real;
      float a[NV];
#pragma unroll
      for (int q = 0; q < NV; ++q) { const float2 t = f2_unpack(acc[q]); a[q] = t.x + t.y; }
      s_loc = lane_transpose_reduce<NV>(a, lane);
#pragma unroll
      for (int q = 0; q < NV; ++q) {
        const float m = __shfl_sync(0xffffffffu, s_loc, q * LPP) * inv_n;
        const float2 t = f2_unpack(acc[q]);
        const float dx = real_x ? t.x - m : 0.f, dy = real_y ? t.y - m : 0.f;
        a[q] = fmaf(dx, dx, dy * dy);
      }
      m2_loc = lane_transpose_reduce<NV>(a, lane);
    }
    PP_MARK(4);
    const int buf = i & 1;
    float2* my_parts = parts + (size_t)(wg * 2 + buf) * PP_MAX_RANKS * NPIX;
    if (!(dbg & 2)) {
      if ((lane % LPP) == 0) {
        const uint32_t la = ptx::smem_u32(my_parts + rank * NPIX + pix);
        const uint32_t lb = bar_parts(buf);
#pragma unroll
        for (int rk = 0; rk < NR; ++rk) ptx::st_async_f32x2(ptx::mapa_shared(la, rk), s_loc, m2_loc, ptx::mapa_shared(lb, rk));
      }
      ptx::mbar_wait_cluster(bar_parts(buf), (uint32_t)((i >> 1) & 1));
    }
    PP_MARK(5);
    // Chan combine of the NR slice partials by the pixel's owner lanes, published to the warp through shared memory
    float2* my_stats = stats + wg * NPIX;
    if ((lane % LPP) == 0) {
      float2 pv[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) pv[r] = my_parts[r * NPIX + pix];
      float tot = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r) tot += pv[r].x;
      const float mean_p = tot / (float)c_real;
      // Chan combine over the real channels: slice r holds n_r = min(64, c_real - 64 r) of them
      float m2 = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        const float n_r = (float)min(CPC, c_real - CPC * r);
        const float d = pv[r].x / n_r - mean_p;
        m2 += fmaf(n_r * d, d, pv[r].y);
      }
      my_stats[pix] = make_float2(mean_p, rsqrtf(m2 / (float)c_real + eps));
    }
    PP_MARK(7);
    // all reads of my_parts done and all stats of the tile visible (the warp only needs its own row, the barrier also
    // orders the re-arm below)
    named_bar_sync(3 + wg, PP_WG_THREADS);
    PP_MARK(8);
    // re-arm this (wg, buffer) barrier for its next use (tile i + 2): strictly before this CTA's own push of tile i + 1,
    // which is what a peer needs before it can push tile i + 2 (see the banner)
    if (tidw == 0 && i + 2 < n_w && !(dbg & 2)) ptx::mbar_arrive_expect_tx(bar_parts(buf), parts_bytes);
    // ---- normalise + affine in packed fp32, bf16x2 out (a warp writes 128 contiguous bytes per pixel) ----
    __nv_bfloat16* orow = R2 ? out + (((long long)b * H + (y0 + rp2)) * W + x0 + xh8) * LDC + c0 + cl
                             : out + (((long long)b * H + (y0 + row0)) * W + x0) * LDC + c0 + cl;
    const float2* srow = R2 ? my_stats + rp2 * TW + xh8 : my_stats + row0 * TW;
    __nv_bfloat16* const orow_next = orow + (long long)W * LDC;   // R2: second output row of this warp
#pragma unroll
    for (int ox_ = 0; ox_ < TW; ++ox_) {
      // R2: values 8..15 are the second row (stats TW entries further, output W pixels further)
      const int ox = R2 ? (ox_ & 7) : ox_;
      if (R2 && ox_ == 8) { orow = orow_next; srow += TW; }
      const float2 st = srow[ox];                                  // broadcast read: (mean, rstd) of this value's pixel
      const f32x2_t cen = f2_sub(acc[ox_], f2_dup(st.x));
      const f32x2_t o2 = f2_fma(f2_mul(cen, f2_dup(st.y)), gw, gb);
      const float2 of = f2_unpack(o2);
      const uint32_t hb = pack_bf16(of.x, of.y);
      if (dbg & 1) { if (of.x == 123.456f) orow[0] = __float2bfloat16(of.y); continue; }
      *reinterpret_cast<uint32_t*>(orow + ox * LDC) = hb;
      if constexpr (SPLIT) {
        const float2 d = f2_unpack(f2_sub(o2, f2_pack(__uint_as_float(hb << 16), __uint_as_float(hb & 0xffff0000u))));
        *reinterpret_cast<uint32_t*>(orow + ox * LDC + C) = pack_bf16(d.x, d.y);
      }
    }
    PP_MARK(6);
  }
#undef PP_MARK
  if constexpr (TRACE) { if (trc) { for (int q = 0; q < 9; ++q) trace[q] = tt[q]; trace[9] = n_w; } }
}

}  // namespace

namespace {

template <int NR, bool SPLIT, bool TRACE, bool R2 = false>
int pp_launch(const CUtensorMap& tmap, const CUtensorMap& tmap_w, const float* bias, const float* ln_w, const float* ln_b,
              __nv_bfloat16* out, int B, int H, int W, int c_real, float eps, int token, cudaStream_t st) {
  auto kfn = dwconv_ln_pp_kernel<NR, SPLIT, TRACE, R2>;
  GDRN_OPT_IN_SMEM(kfn, PP_SMEM);
  const int n_tiles = B * (H / PP_TH) * (W / PP_TW);
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(2 * PP_WG_THREADS);
  cfg.dynamicSmemBytes = PP_SMEM;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = NR;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // see gdrn_launch_dep (common.cuh)
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = gdrn_pdl_enabled() ? 2 : 1;
  // how many clusters of NR one-CTA-per-SM blocks the device can hold at once (GPC-granular), per device
  static int max_clusters[GDRN_MAX_DEVICES] = {};   // (per instantiation: R2 and R1 kernels query separately)
  const int dev = gdrn_cur_device();
  if (max_clusters[dev] == 0) {
    int n = 0;
    cfg.gridDim = dim3(gdrn_num_sms() / NR * NR);
    if (cudaOccupancyMaxActiveClusters(&n, kfn, &cfg) != cudaSuccess || n <= 0) { (void)cudaGetLastError(); n = gdrn_num_sms() / NR / 2; }
    if (n < 1) n = 1;
    max_clusters[dev] = n;
  }
  int nclusters = max_clusters[dev];
  if (nclusters > n_tiles) nclusters = n_tiles;
  cfg.gridDim = dim3(nclusters * NR);
  static long long* d_trace = nullptr;
  if (TRACE && !d_trace) GDRN_CHECK_CUDA(cudaMalloc(&d_trace, 10 * sizeof(long long)));
  long long* trp = TRACE ? d_trace : nullptr;
  GDRN_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kfn, tmap, tmap_w, bias, ln_w, ln_b, out, B, H, W, c_real, eps, token, trp));
  gdrn_count_launch(1);
  if (TRACE) {
    long long h[10];
    GDRN_CHECK_CUDA(cudaMemcpyAsync(h, d_trace, sizeof(h), cudaMemcpyDeviceToHost, st));
    GDRN_CHECK_CUDA(cudaStreamSynchronize(st));
    fprintf(stderr, "[dwconv pp trace] %dx%d C=%d split=%d clusters=%d x %d, wg0 tiles=%lld: tile-wait=%lld token-wait=%lld conv=%lld "
                    "sync+tma=%lld ln-local=%lld push+parts-wait=%lld combine=%lld wg-sync=%lld normalise+store=%lld\n",
            H, W, NR * PP_CPC, (int)SPLIT, nclusters, NR, h[9], h[0], h[1], h[2], h[3], h[4], h[5], h[7], h[8], h[6]);
  }
  return GDRN_OK;
}

}  // namespace

// returns GDRN_OK when launched, 1 when the shape is not handled by this kernel (caller falls back)
int launch_dwconv_ln_pp(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                        __nv_bfloat16* out, int B, int H, int W, int C, float eps, int split, cudaStream_t st, int c_real) {
  if (c_real <= 0) c_real = C;
  if (!(H % PP_TH == 0 && W % PP_TW == 0 && C % PP_CPC == 0)) return 1;
  const int csize = C / PP_CPC;
  if (!(csize == 2 || csize == 3 || csize == 4 || csize == 6 || csize == 8)) return 1;   // the instantiated channel counts
  CUtensorMap tmap, tmap_w;
  {
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[3] = {(uint64_t)C * 4, (uint64_t)W * C * 4, (uint64_t)H * W * C * 4};
    const uint32_t box[4] = {(uint32_t)PP_CPC, (uint32_t)PP_IW, (uint32_t)PP_IH, 1};
    int rc = make_tmap_f32_plain(&tmap, x, 4, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)C, 49};
    const uint64_t str[1] = {(uint64_t)C * 4};
    const uint32_t box[2] = {(uint32_t)PP_CPC, 49};
    int rc = make_tmap_f32_plain(&tmap_w, w49c, 2, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  static int trace_on = -1;  // GDRN_DW_TRACE=1: phase cycle counts of one mid-grid CTA on stderr (synchronises)
  if (trace_on < 0) trace_on = getenv("GDRN_DW_TRACE") ? 1 : 0;
  static int token = -1;     // GDRN_DW_TOKEN=0: no hand-over of the FMA pipe between the warpgroups (measured 3-4 % slower)
  if (token < 0) {
    const char* e = getenv("GDRN_DW_TOKEN");
    token = e ? atoi(e) : 1;
    if (const char* d = getenv("GDRN_DW_DBG")) token = (token & 1) | (atoi(d) & ~7);   // experiment bits, see the kernel
  }
#define PP_ARGS tmap, tmap_w, bias, ln_w, ln_b, out, B, H, W, c_real, eps, token, st
  static int r2 = -1;        // GDRN_DW_R2=0: one output row x 16 pixels per thread in the convolution (the earlier thread tile)
  if (r2 < 0) { const char* e = getenv("GDRN_DW_R2"); r2 = e ? atoi(e) : 1; }
#define PP_CASE(NR)                                                                                    \
  if (csize == NR) {                                                                                   \
    if (trace_on) return split ? pp_launch<NR, true, true>(PP_ARGS) : pp_launch<NR, false, true>(PP_ARGS);   \
    if (r2) return split ? pp_launch<NR, true, false, true>(PP_ARGS) : pp_launch<NR, false, false, true>(PP_ARGS);   \
    return split ? pp_launch<NR, true, false>(PP_ARGS) : pp_launch<NR, false, false>(PP_ARGS);          \
  }
  PP_CASE(2) PP_CASE(3) PP_CASE(4) PP_CASE(6) PP_CASE(8)
#undef PP_CASE
#undef PP_ARGS
  return 1;
}
