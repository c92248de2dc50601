// CUDA-core kernels around the wgmma GEMMs of the dense path: weight repacking, stem patchify,
// ConvNeXt depthwise-7x7 + LayerNorm, LayerNorm + 2x2 patchify, GroupNorm/GELU/bilinear, pose lift.
// Reference semantics: timm 0.6.7 ConvNeXtBlock (third-party), heads/top_down_doublemask_xyz_region_head.py,
// heads/conv_pnp_net.py, core/utils/rot_reps.py:34-55, models/pose_from_pred_centroid_z.py:56-154,
// core/utils/utils.py:31-88.
#include <cooperative_groups.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "dense_ops.h"
#include "dw_helpers.cuh"
#include "gemm_tc.h"

namespace cg = cooperative_groups;

namespace {

// ------------------------------------------------------------------------------------------------
__global__ void pack_kernel(const float* __restrict__ src, void* __restrict__ dst, int dst_is_bf16, PackDesc d) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  // d.lo_delta > 0 (bf16 only): also write lo = bf16(v - float(bf16(v))) at offset + lo_delta (split-bf16 weights)
  const long long total = d.dims[0] * d.dims[1] * d.dims[2] * d.dims[3];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    long long i3 = r % d.dims[3]; r /= d.dims[3];
    long long i2 = r % d.dims[2]; r /= d.dims[2];
    long long i1 = r % d.dims[1]; r /= d.dims[1];
    long long i0 = r;
    float v = src[d.soff + i0 * d.ss[0] + i1 * d.ss[1] + i2 * d.ss[2] + i3 * d.ss[3]];
    long long o = d.doff + i0 * d.ds[0] + i1 * d.ds[1] + i2 * d.ds[2] + i3 * d.ds[3];
    if (dst_is_bf16) {
      const __nv_bfloat16 hi = __float2bfloat16(v);
      reinterpret_cast<__nv_bfloat16*>(dst)[o] = hi;
      if (d.lo_delta > 0) reinterpret_cast<__nv_bfloat16*>(dst)[o + d.lo_delta] = __float2bfloat16(v - __bfloat162float(hi));
    } else {
      reinterpret_cast<float*>(dst)[o] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// stem patchify: one thread per output pixel writes one 128-byte row.
__global__ void stem_patchify_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int H,
                                     int W, int split) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const int OW = W / 4, OH = H / 4;
  const long long total = (long long)B * OH * OW;
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= total) return;
  const int ox = (int)(m % OW);
  const int oy = (int)((m / OW) % OH);
  const int b = (int)(m / ((long long)OW * OH));
  uint4* row = reinterpret_cast<uint4*>(out + m * (split ? 128 : 64));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v[16];
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
      float4 t = *reinterpret_cast<const float4*>(img + (((long long)b * 3 + c) * H + (oy * 4 + ky)) * W + ox * 4);
      v[ky * 4] = t.x; v[ky * 4 + 1] = t.y; v[ky * 4 + 2] = t.z; v[ky * 4 + 3] = t.w;
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      __nv_bfloat162 p0 = __floats2bfloat162_rn(v[j * 8], v[j * 8 + 1]);
      __nv_bfloat162 p1 = __floats2bfloat162_rn(v[j * 8 + 2], v[j * 8 + 3]);
      __nv_bfloat162 p2 = __floats2bfloat162_rn(v[j * 8 + 4], v[j * 8 + 5]);
      __nv_bfloat162 p3 = __floats2bfloat162_rn(v[j * 8 + 6], v[j * 8 + 7]);
      uint4 u;
      u.x = *reinterpret_cast<uint32_t*>(&p0); u.y = *reinterpret_cast<uint32_t*>(&p1);
      u.z = *reinterpret_cast<uint32_t*>(&p2); u.w = *reinterpret_cast<uint32_t*>(&p3);
      row[c * 2 + j] = u;
      if (split) {
        float l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) l[k] = v[j * 8 + k] - __bfloat162float(__float2bfloat16(v[j * 8 + k]));
        uint4 ul;
        ul.x = pack_bf16(l[0], l[1]); ul.y = pack_bf16(l[2], l[3]); ul.z = pack_bf16(l[4], l[5]); ul.w = pack_bf16(l[6], l[7]);
        row[8 + c * 2 + j] = ul;
      }
    }
  }
  row[6] = make_uint4(0, 0, 0, 0);
  row[7] = make_uint4(0, 0, 0, 0);
  if (split) { row[14] = make_uint4(0, 0, 0, 0); row[15] = make_uint4(0, 0, 0, 0); }
}

// ------------------------------------------------------------------------------------------------
// depthwise 7x7 + bias + LayerNorm(C).  Block = 256 threads = S strips x (C/4) channel-quads; a strip is TW
// consecutive output pixels of one image row; a thread owns 4 channels of its strip's TW pixels.
template <int TW>
__global__ void __launch_bounds__(256)
dwconv_ln_kernel(const float* __restrict__ x, const float* __restrict__ w49c, const float* __restrict__ bias,
                 const float* __restrict__ ln_w, const float* __restrict__ ln_b, __nv_bfloat16* __restrict__ out,
                 int B, int H, int W, int C, float eps) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  __shared__ float red[8][TW];  // [warp][pixel]
  const int cq = C >> 2;                 // threads per strip
  const int S = 256 / cq;                // strips per block
  const int strip = threadIdx.x / cq;
  const int c4 = (threadIdx.x % cq) * 4;
  const int strips_per_row = W / TW;
  const long long strip_id = (long long)blockIdx.x * S + strip;  // over B*H*strips_per_row
  const long long n_strips = (long long)B * H * strips_per_row;
  const bool live = strip_id < n_strips;
  const int sx = live ? (int)(strip_id % strips_per_row) : 0;
  const int y = live ? (int)((strip_id / strips_per_row) % H) : 0;
  const int b = live ? (int)(strip_id / ((long long)strips_per_row * H)) : 0;
  const int x0 = sx * TW;

  float4 acc[TW];
  {
    const float4 bv = *reinterpret_cast<const float4*>(bias + c4);
#pragma unroll
    for (int i = 0; i < TW; ++i) acc[i] = bv;
  }
  if (live) {
    for (int ky = 0; ky < 7; ++ky) {
      const int iy = y + ky - 3;
      if (iy < 0 || iy >= H) continue;
      float4 wr[7];
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) wr[kx] = __ldg(reinterpret_cast<const float4*>(w49c + (ky * 7 + kx) * C + c4));
      const float* rowp = x + (((long long)b * H + iy) * W) * C + c4;
#pragma unroll
      for (int j = 0; j < TW + 6; ++j) {
        const int ix = x0 + j - 3;
        if (ix < 0 || ix >= W) continue;
        const float4 v = *reinterpret_cast<const float4*>(rowp + (long long)ix * C);
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const int o = j - kx;  // output pixel index in the strip: ix = x0 + o + kx - 3
          if (o >= 0 && o < TW) {
            acc[o].x = fmaf(v.x, wr[kx].x, acc[o].x);
            acc[o].y = fmaf(v.y, wr[kx].y, acc[o].y);
            acc[o].z = fmaf(v.z, wr[kx].z, acc[o].z);
            acc[o].w = fmaf(v.w, wr[kx].w, acc[o].w);
          }
        }
      }
    }
  }
  // LayerNorm over C: two-pass (mean, then centred variance), reductions over the strip's cq threads.
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wps = cq >> 5;               // warps per strip (1, 2, 4, 8)
  const int w0 = strip * wps;            // first warp of this strip
  float mean[TW];
#pragma unroll
  for (int i = 0; i < TW; ++i) {
    float s = (acc[i].x + acc[i].y) + (acc[i].z + acc[i].w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    mean[i] = s;
  }
  if (wps > 1) {
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < TW; ++i) red[warp][i] = mean[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < TW; ++i) {
      float s = 0.f;
      for (int k = 0; k < wps; ++k) s += red[w0 + k][i];
      mean[i] = s;
    }
    __syncthreads();
  }
  const float invC = 1.0f / (float)C;
  float rstd[TW];
#pragma unroll
  for (int i = 0; i < TW; ++i) {
    mean[i] *= invC;
    float dx = acc[i].x - mean[i], dy = acc[i].y - mean[i], dz = acc[i].z - mean[i], dw = acc[i].w - mean[i];
    float s = (dx * dx + dy * dy) + (dz * dz + dw * dw);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    rstd[i] = s;
  }
  if (wps > 1) {
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < TW; ++i) red[warp][i] = rstd[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < TW; ++i) {
      float s = 0.f;
      for (int k = 0; k < wps; ++k) s += red[w0 + k][i];
      rstd[i] = s;
    }
  }
  if (!live) return;
  const float4 gw = *reinterpret_cast<const float4*>(ln_w + c4);
  const float4 gb = *reinterpret_cast<const float4*>(ln_b + c4);
  __nv_bfloat16* orow = out + ((((long long)b * H + y) * W) + x0) * C + c4;
#pragma unroll
  for (int i = 0; i < TW; ++i) {
    const float r = rsqrtf(rstd[i] * invC + eps);
    float o0 = fmaf((acc[i].x - mean[i]) * r, gw.x, gb.x);
    float o1 = fmaf((acc[i].y - mean[i]) * r, gw.y, gb.y);
    float o2 = fmaf((acc[i].z - mean[i]) * r, gw.z, gb.z);
    float o3 = fmaf((acc[i].w - mean[i]) * r, gw.w, gb.w);
    __nv_bfloat162 p0 = __floats2bfloat162_rn(o0, o1), p1 = __floats2bfloat162_rn(o2, o3);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&p0);
    u.y = *reinterpret_cast<uint32_t*>(&p1);
    *reinterpret_cast<uint2*>(orow + (long long)i * C) = u;
  }
}


// ------------------------------------------------------------------------------------------------
// depthwise 7x7 + bias + LayerNorm(C), thread-block-cluster + packed-FP32 version (the one the forward uses).
//   CTA  = one TW x TH output tile of one image x CPC channels (16x8 x 64 ch, two CTAs per SM so that one CTA's tile
//          load overlaps the other's arithmetic; 8x8 x 128 ch for 8x8 images).  The zero-padded (TW+6)x(TH+6) x CPC
//          fp32 input tile is fetched by ONE TMA box load (halo = out-of-bounds zero fill).
//   thread = a PAIR of adjacent channels x one output row (TW pixels).  All arithmetic is fma.rn.f32x2
//          (f2_* element pairs, the same IEEE operation per lane); the input pairs
//          and the filter pairs are 8-byte shared-memory loads, conflict-free with lanes = channel pairs.
//   cluster = the C/CPC CTAs (2/4/8) that together hold all channels of the tile: the LayerNorm statistics are
//          combined across them through distributed shared memory with ONE cluster barrier (see below).
// In-warp per-pixel channel sums use a transposing shuffle reduction.
// Depthwise 7x7 + bias + LayerNorm(C) -> bf16 GEMM operand.  One CTA = (TW x TH pixel tile) x CPC channels of one
// image; the CTAs of a cluster hold the C / CPC channel slices of the same tile.  A thread owns one channel PAIR
// (packed fma.rn.f32x2) and R consecutive output rows x TW pixels.  It walks the R + 6 input rows once: each row is
// loaded from shared memory a single time (TW + 6 LDS.64) and applied to every output row it contributes to, and
// the filter row fetched for output row r is kept in registers for output row r + 1 of the next step, so that one
// step costs TW + 6 + 7 shared-memory loads for R * 7 * TW packed FMAs (R = 2: 0.13 loads per FMA instead of 0.26;
// the R = 1 form was co-limited by shared-memory bandwidth, see profiles/).
template <int TW, int TH, int CPC, int R, int MINB>
__global__ void __launch_bounds__((CPC / 2) * TH / R, MINB)
dwconv_ln_cluster_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                         const float* __restrict__ bias, const float* __restrict__ ln_w,
                         const float* __restrict__ ln_b, __nv_bfloat16* __restrict__ out, int B, int H, int W, int C,
                         int c_real, float eps, int split, long long* trace) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  static_assert(R == 1 || R == 2, "rows per thread");
  const bool trc = trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == B / 2 && threadIdx.x == 0;
  long long tt[6];
  if (trc) tt[0] = clock64();
  constexpr int PAIRS = CPC / 2;              // channel pairs = threads per thread-row (CPC = channels per CTA)
  constexpr int IW = TW + 6;
  constexpr int IH = TH + 6;
  constexpr int NPIX = TW * TH;
  constexpr int WPR = PAIRS / 32;             // warps per thread-row
  constexpr int NV = R * TW;                  // pixels per thread
  constexpr int LPP = 32 / NV;                // lanes per pixel after the transposing reduction (1, 2 or 4)
  static_assert(NV == 8 || NV == 16 || NV == 32, "pixels per thread");
  extern __shared__ __align__(1024) float smem_dw[];   // TMA destination first: 128-byte aligned
  float* tile = smem_dw;                      // [IH][IW][CPC]
  float* wsm = tile + IH * IW * CPC;          // [49][CPC]
  float2* s_parts = reinterpret_cast<float2*>(wsm + 49 * CPC);  // [8 ranks * WPR][NPIX] (sum, M2) partials, pushed by peers
  unsigned long long* tma_bar_p = reinterpret_cast<unsigned long long*>(s_parts + 8 * WPR * NPIX);   // [0] TMA, [1] partials

  cg::cluster_group cluster = cg::this_cluster();
  const int nrank = (int)cluster.num_blocks();
  const int c0 = blockIdx.x * CPC;
  const int tiles_x = W / TW;
  const int x0 = (blockIdx.y % tiles_x) * TW;
  const int y0 = (blockIdx.y / tiles_x) * TH;
  const int b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31;
  const int pair = tid % PAIRS;
  const int row0 = (tid / PAIRS) * R;         // first output row of this thread
  const int wc = (tid >> 5) % WPR;            // which 64-channel group of the CTA this warp holds
  const int cl = 2 * pair;                    // first channel of the pair (CTA-local)

  const uint32_t bar = ptx::smem_u32(tma_bar_p);
  const uint32_t parts_bar = bar + 8;
  if (tid == 0) {
    ptx::mbar_init(bar, 1);
    ptx::mbar_init(parts_bar, 1);
    ptx::fence_barrier_init();
    // every (rank, 64-channel warp group, pixel) partial of the cluster lands here as one 8-byte st.async
    ptx::mbar_arrive_expect_tx(parts_bar, (uint32_t)(nrank * WPR * NPIX * sizeof(float2)));
  }
  __syncthreads();
  if (tid == 0) {
    ptx::mbar_arrive_expect_tx(bar, (uint32_t)((IH * IW + 49) * CPC * sizeof(float)));
    ptx::tma_load_2d(ptx::smem_u32(wsm), &tmap_w, bar, c0, 0);          // this CTA's 49 x CPC filter taps
    ptx::tma_load_4d(ptx::smem_u32(tile), &tmap_x, bar, c0, x0 - 3, y0 - 3, b);
  }
  // split-phase cluster barrier: "my barriers exist" is announced here and only waited for right before the push
  // (a conv later), so the start-up skew between the CTAs of a cluster is off the critical path
  asm volatile("barrier.cluster.arrive.release;" ::: "memory");
  f32x2_t acc[R][TW];
  {
    const f32x2_t bv = f2_pack(__ldg(bias + c0 + cl), __ldg(bias + c0 + cl + 1));
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int i = 0; i < TW; ++i) acc[r][i] = bv;
  }
  ptx::mbar_wait(bar, 0);    // filter taps + input tile landed
  if (trc) tt[1] = clock64();

  // ---- convolution: input row i feeds output row r with filter row ky = i - r ----
  {
    f32x2_t wprev[7];
#pragma unroll
    for (int i = 0; i < R + 6; ++i) {
      f32x2_t v[IW], wk[7];
      const float* rowp = tile + ((row0 + i) * IW) * CPC + cl;
#pragma unroll
      for (int j = 0; j < IW; ++j) v[j] = *reinterpret_cast<const f32x2_t*>(rowp + j * CPC);
      if (i < 7) {
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) wk[kx] = *reinterpret_cast<const f32x2_t*>(wsm + (i * 7 + kx) * CPC + cl);
#pragma unroll
        for (int kx = 0; kx < 7; ++kx)
#pragma unroll
          for (int ox = 0; ox < TW; ++ox) acc[0][ox] = f2_fma(v[ox + kx], wk[kx], acc[0][ox]);
      }
      if (R == 2 && i >= 1) {
#pragma unroll
        for (int kx = 0; kx < 7; ++kx)
#pragma unroll
          for (int ox = 0; ox < TW; ++ox) acc[R - 1][ox] = f2_fma(v[ox + kx], wprev[kx], acc[R - 1][ox]);
      }
      if (R == 2 && i < 7) {
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) wprev[kx] = wk[kx];
      }
    }
  }
  if (trc) tt[2] = clock64();
  float ax[NV], ay[NV];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < TW; ++i) { const float2 t = f2_unpack(acc[r][i]); ax[r * TW + i] = t.x; ay[r * TW + i] = t.y; }

  // ---- LayerNorm over all C channels of each pixel ----
  // A warp holds 64 channels of its NV pixels: it computes (sum, M2 about its own mean) per pixel with
  // shuffles only, PUSHES that partial into every CTA of the cluster (distributed shared memory stores), and after
  // ONE cluster barrier each warp combines the C/64 partials with Chan's parallel-variance formula.  No block-level
  // barrier, no remote loads, and nothing remote is touched after the barrier (so no exit barrier is needed).
  // Zero pad channels (c >= c_real, all in the last 64-channel group) are left out of the group's mean and M2.
  const int pix = row0 * TW + lane / LPP;   // the thread's R rows are contiguous in the row-major tile
  float s_loc, m2_loc;
  {
    const int cw = c0 + wc * 64;             // first channel of this warp's group
    const float inv_n = 1.0f / (float)min(64, c_real - cw);
    const bool real_x = c0 + cl < c_real, real_y = c0 + cl + 1 < c_real;
    float a[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) a[i] = ax[i] + ay[i];
    s_loc = lane_transpose_reduce<NV>(a, lane);           // lane L: pixel L / LPP of this thread-row
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float m = __shfl_sync(0xffffffffu, s_loc, i * LPP) * inv_n;
      const float dx = real_x ? ax[i] - m : 0.f, dy = real_y ? ay[i] - m : 0.f;
      a[i] = fmaf(dx, dx, dy * dy);
    }
    m2_loc = lane_transpose_reduce<NV>(a, lane);
  }
  const int nparts = nrank * WPR;
  asm volatile("barrier.cluster.wait.acquire;" ::: "memory");   // every peer has initialised its partials barrier
  {
    const int part = (int)cluster.block_rank() * WPR + wc;
    if ((lane % LPP) == 0) {
      // push with st.async: the 8 bytes complete transaction bytes on the peer's barrier, so there is no fence and no
      // cluster-wide rendezvous -- a CTA continues as soon as ITS partials are in, stragglers only delay themselves
      const uint32_t la = ptx::smem_u32(s_parts + part * NPIX + pix);
      for (int rk = 0; rk < nrank; ++rk)
        ptx::st_async_f32x2(ptx::mapa_shared(la, rk), s_loc, m2_loc, ptx::mapa_shared(parts_bar, rk));
    }
  }
  if (trc) tt[3] = clock64();
  ptx::mbar_wait_cluster(parts_bar, 0);
  if (trc) tt[4] = clock64();
  float mean_p, rstd_p;
  {
    float tot = 0.f;
    for (int k = 0; k < nparts; ++k) tot += s_parts[k * NPIX + pix].x;
    mean_p = tot / (float)c_real;
    // Chan combine over the real channels: group k holds n_k = min(64, c_real - 64 k) of them
    float m2 = 0.f;
    for (int k = 0; k < nparts; ++k) {
      const float2 v = s_parts[k * NPIX + pix];
      const float n_k = (float)min(64, c_real - 64 * k);
      const float d = v.x / n_k - mean_p;
      m2 += fmaf(n_k * d, d, v.y);
    }
    rstd_p = rsqrtf(m2 / (float)c_real + eps);
  }
  // ---- normalise + affine, bf16x2 out (a warp writes 128 contiguous bytes per pixel) ----
  const float gw0 = __ldg(ln_w + c0 + cl), gw1 = __ldg(ln_w + c0 + cl + 1);
  const float gb0 = __ldg(ln_b + c0 + cl), gb1 = __ldg(ln_b + c0 + cl + 1);
  const int ldc = split ? 2 * C : C;  // split mode: rows are [hi C | lo C]
#pragma unroll
  for (int r = 0; r < R; ++r) {
    __nv_bfloat16* orow = out + (((long long)b * H + (y0 + row0 + r)) * W + x0) * ldc + c0 + cl;
#pragma unroll
    for (int ox = 0; ox < TW; ++ox) {
      const int i = r * TW + ox;
      const float m = __shfl_sync(0xffffffffu, mean_p, i * LPP);
      const float rs = __shfl_sync(0xffffffffu, rstd_p, i * LPP);
      const float o0 = fmaf((ax[i] - m) * rs, gw0, gb0), o1 = fmaf((ay[i] - m) * rs, gw1, gb1);
      const __nv_bfloat162 o = __floats2bfloat162_rn(o0, o1);
      *reinterpret_cast<__nv_bfloat162*>(orow + (long long)ox * ldc) = o;
      if (split) {
        const float2 of = __bfloat1622float2(o);
        *reinterpret_cast<__nv_bfloat162*>(orow + (long long)ox * ldc + C) = __floats2bfloat162_rn(o0 - of.x, o1 - of.y);
      }
    }
  }
  if (trc) {
    tt[5] = clock64();
    for (int i = 0; i < 5; ++i) trace[i] = tt[i + 1] - tt[i];
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm2d + 2x2 stride-2 patchify (ConvNeXt downsample front half).  One warp per OUTPUT pixel: it loads the four
// source pixels of the 2x2 patch up front (4 x C fp32 in flight per warp -- the one-pixel-per-warp form was latency
// bound at 1.4 TB/s), normalises each over its C channels with interleaved shuffle reductions, and writes the
// patch row [p00 C | p01 C | p10 C | p11 C] (bf16, plus the lo halves in split mode).  C = 128 * NV.
template <int NV, int VW>
__global__ void __launch_bounds__(256)
ln_patchify2_kernel(const float* __restrict__ x, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                    __nv_bfloat16* __restrict__ out, int B, int H, int W, float eps, int split, int c_real) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  // C = 32 * VW * NV: lane owns VW consecutive channels of every 32 * VW-channel group (VW = 4: C % 128 == 0; VW = 2: C % 64 == 0)
  constexpr int C = 32 * VW * NV;
  const int OW = W / 2, OH = H / 2;
  const long long m2 = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (m2 >= (long long)B * OH * OW) return;
  const int lane = threadIdx.x & 31;
  const int ox = (int)(m2 % OW);
  const int oy = (int)((m2 / OW) % OH);
  const int b = (int)(m2 / ((long long)OW * OH));
  float v[4][NV][VW];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const float* src = x + (((long long)b * H + (2 * oy + (p >> 1))) * W + (2 * ox + (p & 1))) * C;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if constexpr (VW == 4) {
        const float4 t = *reinterpret_cast<const float4*>(src + (k * 32 + lane) * 4);
        v[p][k][0] = t.x; v[p][k][1] = t.y; v[p][k][2] = t.z; v[p][k][3] = t.w;
      } else {
        const float2 t = *reinterpret_cast<const float2*>(src + (k * 32 + lane) * 2);
        v[p][k][0] = t.x; v[p][k][1] = t.y;
      }
    }
  }
  float s[4], q[4];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    s[p] = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if constexpr (VW == 4) s[p] += (v[p][k][0] + v[p][k][1]) + (v[p][k][2] + v[p][k][3]);
      else s[p] += v[p][k][0] + v[p][k][1];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int p = 0; p < 4; ++p) s[p] += __shfl_xor_sync(0xffffffffu, s[p], o);
  // centred sum of squares over the c_real real channels only: the zero pad channels are masked out of the pass
  // (subtracting their (C - c_real) * mean^2 afterwards cancels catastrophically when |mean| >> std)
  auto centred = [c_real](float x, float mean, int c) { return c < c_real ? x - mean : 0.f; };
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    s[p] = s[p] / (float)c_real;   // mean (zero pad channels do not contribute to the sum)
    q[p] = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int c = (k * 32 + lane) * VW;
      if constexpr (VW == 4) {
        const float dx = centred(v[p][k][0], s[p], c), dy = centred(v[p][k][1], s[p], c + 1);
        const float dz = centred(v[p][k][2], s[p], c + 2), dw = centred(v[p][k][3], s[p], c + 3);
        q[p] += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      } else {
        const float dx = centred(v[p][k][0], s[p], c), dy = centred(v[p][k][1], s[p], c + 1);
        q[p] += dx * dx + dy * dy;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int p = 0; p < 4; ++p) q[p] += __shfl_xor_sync(0xffffffffu, q[p], o);
  __nv_bfloat16* dst = out + m2 * ((split ? 8LL : 4LL) * C);
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = (k * 32 + lane) * VW;
    float gw[VW], gb[VW];
    if constexpr (VW == 4) {
      const float4 w4 = *reinterpret_cast<const float4*>(ln_w + c), b4 = *reinterpret_cast<const float4*>(ln_b + c);
      gw[0] = w4.x; gw[1] = w4.y; gw[2] = w4.z; gw[3] = w4.w; gb[0] = b4.x; gb[1] = b4.y; gb[2] = b4.z; gb[3] = b4.w;
    } else {
      const float2 w2 = *reinterpret_cast<const float2*>(ln_w + c), b2 = *reinterpret_cast<const float2*>(ln_b + c);
      gw[0] = w2.x; gw[1] = w2.y; gb[0] = b2.x; gb[1] = b2.y;
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float r = rsqrtf(q[p] / (float)c_real + eps);
      float o[VW];
#pragma unroll
      for (int e = 0; e < VW; ++e) o[e] = fmaf((v[p][k][e] - s[p]) * r, gw[e], gb[e]);
      uint32_t hw[VW / 2], lw[VW / 2];
#pragma unroll
      for (int e = 0; e < VW; e += 2) {
        const __nv_bfloat162 h2 = __floats2bfloat162_rn(o[e], o[e + 1]);
        const float2 f = __bfloat1622float2(h2);
        hw[e / 2] = *reinterpret_cast<const uint32_t*>(&h2);
        lw[e / 2] = pack_bf16(o[e] - f.x, o[e + 1] - f.y);
      }
      __nv_bfloat16* dh = dst + p * C + c;
      __nv_bfloat16* dl = dst + 4LL * C + p * C + c;      // lo half of the [hi 4C | lo 4C] row
      if constexpr (VW == 4) {
        *reinterpret_cast<uint2*>(dh) = make_uint2(hw[0], hw[1]);
        if (split) *reinterpret_cast<uint2*>(dl) = make_uint2(lw[0], lw[1]);
      } else {
        *reinterpret_cast<uint32_t*>(dh) = hw[0];
        if (split) *reinterpret_cast<uint32_t*>(dl) = lw[0];
      }
    }
  }
}

__device__ __forceinline__ void load8(const void* raw, int is_f32, long long off, float (&v)[8]) {
  if (is_f32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(raw) + off);
    float4 a = p[0], b = p[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(raw) + off);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 f = __bfloat1622float2(h[k]);
      v[2 * k] = f.x; v[2 * k + 1] = f.y;
    }
  }
}

// 8 consecutive channels -> bf16 (hi) at dst, and, in split mode, lo = bf16(v - hi) at dst + lo_off
__device__ __forceinline__ void store8_split(__nv_bfloat16* dst, const float (&o)[8], int split, long long lo_off) {
  uint4 u;
  u.x = pack_bf16(o[0], o[1]); u.y = pack_bf16(o[2], o[3]); u.z = pack_bf16(o[4], o[5]); u.w = pack_bf16(o[6], o[7]);
  *reinterpret_cast<uint4*>(dst) = u;
  if (split) {
    float l[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) l[k] = o[k] - __bfloat162float(__float2bfloat16(o[k]));
    u.x = pack_bf16(l[0], l[1]); u.y = pack_bf16(l[2], l[3]); u.z = pack_bf16(l[4], l[5]); u.w = pack_bf16(l[6], l[7]);
    *reinterpret_cast<uint4*>(dst + lo_off) = u;
  }
}

__global__ void cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n;
       i += (long long)gridDim.x * blockDim.x * 4) {
    if (i + 3 < n) {
      float4 v = *reinterpret_cast<const float4*>(src + i);
      __nv_bfloat162 p0 = __floats2bfloat162_rn(v.x, v.y), p1 = __floats2bfloat162_rn(v.z, v.w);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&p0);
      u.y = *reinterpret_cast<uint32_t*>(&p1);
      *reinterpret_cast<uint2*>(dst + i) = u;
    } else {
      for (long long j = i; j < n; ++j) dst[j] = __float2bfloat16(src[j]);
    }
  }
}

// fp32 [rows, C] -> split bf16 [rows, 2C] = [hi C | lo C]
__global__ void cast_split_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long rows, int C) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const long long total = rows * (C / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (C / 8);
    const int c8 = (int)(i % (C / 8)) * 8;
    float v[8];
    load8(src, 1, r * C + c8, v);
    store8_split(dst + r * 2 * C + c8, v, 1, C);
  }
}

__global__ void bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long n) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = __bfloat162float(src[i]);
}

// split bf16 [rows, 2C] = [hi C | lo C] -> fp32 [rows, C] = hi + lo
__global__ void split_to_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long rows, int C) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * C; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C, c = i % C;
    dst[i] = __bfloat162float(src[r * 2 * C + c]) + __bfloat162float(src[r * 2 * C + C + c]);
  }
}

// ------------------------------------------------------------------------------------------------
// GroupNorm apply + exact-erf GELU (+ bilinear x2, align_corners=True).  One thread per (output pixel, 8 channels).
// per-(image, group) mean / rstd from the double sums accumulated by the conv epilogue
__global__ void gn_finalize_kernel(const double* __restrict__ stats, float2* __restrict__ mr, int n_bg, double count,
                                   float eps) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_bg) return;
  const double mean = stats[2 * i] / count;
  double var = stats[2 * i + 1] / count - mean * mean;
  if (var < 0.0) var = 0.0;
  mr[i] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
}

// GroupNorm apply + GELU: one thread per (4 consecutive pixels, 8 channels); the per-channel scale/shift is
// computed once per thread, GELU uses the packed-half2 tanh.approx form (two elements per instruction).
constexpr int GN_PPT = 4;
__global__ void __launch_bounds__(256)
gn_gelu_kernel(const void* __restrict__ raw, int raw_is_f32, const double* __restrict__ stats, double count, float eps,
               const float* __restrict__ gn_w, const float* __restrict__ gn_b, __nv_bfloat16* __restrict__ out, int B,
               int hw, int C, int groups, int split) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const int cv = C >> 3;
  const unsigned total = (unsigned)B * (hw / GN_PPT) * cv;  // < 2^31 (checked by the launcher)
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  // per-(image, group) mean / rstd of the (at most two) images this block touches, from the double sums accumulated by the
  // conv epilogue -- the arithmetic of gn_finalize_kernel, folded in here to save one launch per GroupNorm
  __shared__ float2 mr_s[2][32];
  const int b_first = (int)((blockIdx.x * blockDim.x / (unsigned)cv) / (unsigned)(hw / GN_PPT));
  if ((int)threadIdx.x < 2 * groups) {
    const int bi = (int)threadIdx.x / groups, g = (int)threadIdx.x % groups;
    if (b_first + bi < B) {
      const long long i = (long long)(b_first + bi) * groups + g;
      const double mean = stats[2 * i] / count;
      double var = stats[2 * i + 1] / count - mean * mean;
      if (var < 0.0) var = 0.0;
      mr_s[bi][g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
  }
  __syncthreads();
  if (idx >= total) return;
  const int c8 = (int)(idx % (unsigned)cv) * 8;
  const unsigned pg = idx / (unsigned)cv;                  // pixel group over all images
  const int b = (int)(pg / (unsigned)(hw / GN_PPT));
  const long long pix0 = (long long)pg * GN_PPT;           // first pixel (global index over B*hw)
  const int cpg = C / groups;
  float a[8], s[8];
  {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(gn_w + c8)), w1 = __ldg(reinterpret_cast<const float4*>(gn_w + c8 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(gn_b + c8)), b1 = __ldg(reinterpret_cast<const float4*>(gn_b + c8 + 4));
    const float gw[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    const float gb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    const float2* mrow = mr_s[b - b_first];
    float2 m = mrow[c8 / cpg];
    int gcur = c8 / cpg;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int g = (c8 + k) / cpg;
      if (g != gcur) { m = mrow[g]; gcur = g; }
      a[k] = m.y * gw[k];
      s[k] = fmaf(-m.x, a[k], gb[k]);
    }
  }
  float v[GN_PPT][8];
#pragma unroll
  for (int i = 0; i < GN_PPT; ++i) load8(raw, raw_is_f32, (pix0 + i) * C + c8, v[i]);
  if (split) {  // split-bf16 (x3) mode: exact-erf GELU, [hi C | lo C] rows
#pragma unroll
    for (int i = 0; i < GN_PPT; ++i) {
      float o[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = gelu_erf(fmaf(v[i][k], a[k], s[k]));
      store8_split(out + (pix0 + i) * 2 * C + c8, o, 1, C);
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < GN_PPT; ++i) {
    uint4 u;
    u.x = gelu_pack2_f16(fmaf(v[i][0], a[0], s[0]), fmaf(v[i][1], a[1], s[1]));
    u.y = gelu_pack2_f16(fmaf(v[i][2], a[2], s[2]), fmaf(v[i][3], a[3], s[3]));
    u.z = gelu_pack2_f16(fmaf(v[i][4], a[4], s[4]), fmaf(v[i][5], a[5], s[5]));
    u.w = gelu_pack2_f16(fmaf(v[i][6], a[6], s[6]), fmaf(v[i][7], a[7], s[7]));
    *reinterpret_cast<uint4*>(out + (pix0 + i) * C + c8) = u;
  }
}

// GroupNorm apply + exact GELU -> fp32 (feeds the fp32 FC stack of the split-bf16 mode)
__global__ void gn_gelu_f32_kernel(const float* __restrict__ raw, const float2* __restrict__ mr,
                                   const float* __restrict__ gn_w, const float* __restrict__ gn_b,
                                   float* __restrict__ out, int B, int hw, int C, int groups) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const long long total = (long long)B * hw * C;
  const int cpg = C / groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int b = (int)(i / ((long long)hw * C));
    const float2 m = mr[(long long)b * groups + c / cpg];
    out[i] = gelu_erf((raw[i] - m.x) * m.y * gn_w[c] + gn_b[c]);
  }
}

// y[b, n] = act(sum_k x[b,k] * W[n,k] + bias[n]) in fp32 on the CUDA cores (Patch-PnP FC stack of the split-bf16 mode:
// conv_pnp_net.py:150-183 fc1 8192 -> 1024, fc2 -> 256, fc_r | fc_t -> 16).  The op is bound by streaming W (fc1: 32 MB) once,
// so it is split along K over the whole chip: block = FC_NB neurons x BT batch rows x one K slice; x and W tiles of FC_KT
// k-values are staged through shared memory in [k][row] layout (the global loads of the next tile are in flight during the
// FMAs of the current one), a thread owns 4 neurons x BT/16 rows.  The slices' partial sums go to part[ks][b][n];
// fc_f32_reduce_kernel adds them in slice order, then bias and GELU: deterministic, no atomics.  (The previous forms -- one
// output per warp, then 4 neurons x 16 rows per warp straight from global memory -- re-read x or W from L2 hundreds of times:
// 150 / 480 us for fc1 at B = 64.)
constexpr int FC_NB = 64, FC_KT = 32, FC_MAX_KS = 32;
template <int BT>
__global__ void __launch_bounds__(256)
fc_f32_partial_kernel(const float* __restrict__ x, const float* __restrict__ W, float* __restrict__ part, int B, int N, int K,
                      int kslice) {
  constexpr int RB = BT / 16;                       // batch rows per thread
  __shared__ __align__(16) float xs[FC_KT][BT];
  __shared__ __align__(16) float ws[FC_KT][FC_NB];
  ptx::griddep_launch();
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int n0 = blockIdx.x * FC_NB, ks = blockIdx.y, b0 = blockIdx.z * BT;
  const int kbeg = ks * kslice;
  // loader mapping: rows vary fastest inside a warp (conflict-free transposing stores), 8 k-quads per row
  const int lrow = t & 31, lkq = t >> 5;
  const bool w_ok0 = n0 + lrow < N, w_ok1 = n0 + lrow + 32 < N;
  const float* wp0 = W + (long long)(n0 + lrow) * K + kbeg + lkq * 4;
  const float* wp1 = wp0 + 32LL * K;
  // x rows: BT = 64 -> two passes of 32 rows; BT = 16 -> threads 0..127 (16 rows x 8 k-quads)
  const int xrow = BT == 64 ? lrow : (t & 15), xkq = BT == 64 ? lkq : ((t >> 4) & 7);
  const bool x_act = BT == 64 || t < 128;
  const bool x_ok0 = x_act && b0 + xrow < B, x_ok1 = BT == 64 && b0 + xrow + 32 < B;
  const float* xp0 = x + (long long)(b0 + xrow) * K + kbeg + xkq * 4;
  const float* xp1 = xp0 + 32LL * K;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  ptx::griddep_wait();
  float4 rw0 = w_ok0 ? __ldg(reinterpret_cast<const float4*>(wp0)) : z4;
  float4 rw1 = w_ok1 ? __ldg(reinterpret_cast<const float4*>(wp1)) : z4;
  float4 rx0 = x_ok0 ? *reinterpret_cast<const float4*>(xp0) : z4;
  float4 rx1 = x_ok1 ? *reinterpret_cast<const float4*>(xp1) : z4;
  float acc[RB][4];
#pragma unroll
  for (int i = 0; i < RB; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int ntiles = kslice / FC_KT;
  for (int kt = 0; kt < ntiles; ++kt) {
    __syncthreads();   // the previous tile has been consumed
    ws[lkq * 4 + 0][lrow] = rw0.x; ws[lkq * 4 + 1][lrow] = rw0.y; ws[lkq * 4 + 2][lrow] = rw0.z; ws[lkq * 4 + 3][lrow] = rw0.w;
    ws[lkq * 4 + 0][lrow + 32] = rw1.x; ws[lkq * 4 + 1][lrow + 32] = rw1.y; ws[lkq * 4 + 2][lrow + 32] = rw1.z; ws[lkq * 4 + 3][lrow + 32] = rw1.w;
    if (x_act) {
      xs[xkq * 4 + 0][xrow] = rx0.x; xs[xkq * 4 + 1][xrow] = rx0.y; xs[xkq * 4 + 2][xrow] = rx0.z; xs[xkq * 4 + 3][xrow] = rx0.w;
      if (BT == 64) {
        xs[xkq * 4 + 0][(xrow + 32) % BT] = rx1.x; xs[xkq * 4 + 1][(xrow + 32) % BT] = rx1.y;
        xs[xkq * 4 + 2][(xrow + 32) % BT] = rx1.z; xs[xkq * 4 + 3][(xrow + 32) % BT] = rx1.w;
      }
    }
    __syncthreads();
    if (kt + 1 < ntiles) {   // next tile: in flight during the FMAs below
      const int o = (kt + 1) * FC_KT;
      rw0 = w_ok0 ? __ldg(reinterpret_cast<const float4*>(wp0 + o)) : z4;
      rw1 = w_ok1 ? __ldg(reinterpret_cast<const float4*>(wp1 + o)) : z4;
      rx0 = x_ok0 ? *reinterpret_cast<const float4*>(xp0 + o) : z4;
      rx1 = x_ok1 ? *reinterpret_cast<const float4*>(xp1 + o) : z4;
    }
#pragma unroll
    for (int k = 0; k < FC_KT; ++k) {
      const float4 wv = *reinterpret_cast<const float4*>(&ws[k][tx * 4]);
      float a[RB];
      if constexpr (RB == 4) {
        const float4 av = *reinterpret_cast<const float4*>(&xs[k][ty * 4]);
        a[0] = av.x; a[1] = av.y; a[2] = av.z; a[3] = av.w;
      } else {
#pragma unroll
        for (int i = 0; i < RB; ++i) a[i] = xs[k][ty * RB + i];
      }
#pragma unroll
      for (int i = 0; i < RB; ++i) {
        acc[i][0] = fmaf(a[i], wv.x, acc[i][0]); acc[i][1] = fmaf(a[i], wv.y, acc[i][1]);
        acc[i][2] = fmaf(a[i], wv.z, acc[i][2]); acc[i][3] = fmaf(a[i], wv.w, acc[i][3]);
      }
    }
  }
  const int n = n0 + tx * 4;
  if (n < N) {
#pragma unroll
    for (int i = 0; i < RB; ++i) {
      const int b = b0 + ty * RB + i;
      if (b < B)
        *reinterpret_cast<float4*>(part + ((long long)ks * B + b) * N + n) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
  }
}

// y[b, n] = act(bias[n] + sum over the K slices, in slice order)
__global__ void __launch_bounds__(256)
fc_f32_reduce_kernel(const float* __restrict__ part, const float* __restrict__ bias, float* __restrict__ y, int B, int N, int ks_n,
                     int ldy, int gelu) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // one float4 of outputs
  const int nq = N >> 2;
  if (i >= B * nq) return;
  const int b = i / nq, n = (i - b * nq) * 4;
  float4 s = *reinterpret_cast<const float4*>(part + (long long)b * N + n);
  for (int ks = 1; ks < ks_n; ++ks) {
    const float4 v = *reinterpret_cast<const float4*>(part + ((long long)ks * B + b) * N + n);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + n));
  s.x += bv.x; s.y += bv.y; s.z += bv.z; s.w += bv.w;
  if (gelu) { s.x = gelu_erf(s.x); s.y = gelu_erf(s.y); s.z = gelu_erf(s.z); s.w = gelu_erf(s.w); }
  float* yr = y + (long long)b * ldy + n;
  yr[0] = s.x; yr[1] = s.y; yr[2] = s.z; yr[3] = s.w;
}

// nn.UpsamplingBilinear2d(scale_factor=2) (align_corners=True) on NHWC bf16: src = dst * (in-1)/(out-1)
// (top_down_doublemask_xyz_region_head.py:99-104).  A thread produces a 2 x 2 block of output pixels x 8 channels: the four
// outputs read from a window of (2 + DY) x (2 + DX) input pixels (the source step is < 0.5, so neighbouring outputs start at
// the same or the next input pixel: DY, DX in {0, 1}, uniform over the warp), 4 - 9 pixel loads per block instead of 16.
// Per output the arithmetic is the one-pixel-per-thread form's: o = w00*v00 + w01*v01 + w10*v10 + w11*v11.
template <int DY, int DX>
__device__ __forceinline__ void upsample_block(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int b, int h,
                                               int w, int C, int split, int ldc, int c8, int oy0, int ox0, const int (&y0)[2],
                                               const int (&x0)[2], const float (&ly)[2], const float (&lx)[2]) {
  float win[2 + DY][2 + DX][8];
#pragma unroll
  for (int r = 0; r < 2 + DY; ++r)
#pragma unroll
    for (int c = 0; c < 2 + DX; ++c) {
      const long long off = (((long long)b * h + min(y0[0] + r, h - 1)) * w + min(x0[0] + c, w - 1)) * ldc + c8;
      load8(in, 0, off, win[r][c]);
      if (split) {  // value = hi + lo
        float t[8];
        load8(in, 0, off + C, t);
#pragma unroll
        for (int k = 0; k < 8; ++k) win[r][c][k] += t[k];
      }
    }
  const int oh = 2 * h, ow = 2 * w;
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int wr = r * DY, wc = c * DX;   // window position of this output's (y0, x0)
      const float w00 = (1.f - ly[r]) * (1.f - lx[c]), w01 = (1.f - ly[r]) * lx[c], w10 = ly[r] * (1.f - lx[c]), w11 = ly[r] * lx[c];
      float o[8];
#pragma unroll
      for (int k = 0; k < 8; ++k)
        o[k] = w00 * win[wr][wc][k] + w01 * win[wr][wc + 1][k] + w10 * win[wr + 1][wc][k] + w11 * win[wr + 1][wc + 1][k];
      store8_split(out + (((long long)b * oh + oy0 + r) * ow + ox0 + c) * ldc + c8, o, split, C);
    }
}

__global__ void __launch_bounds__(256)
upsample2x_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int B, int h, int w, int C,
                  int split) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const int cv = C >> 3;
  const int oh = 2 * h, ow = 2 * w;
  const unsigned total = (unsigned)B * h * w * cv;       // one thread per 2 x 2 output block and 8 channels
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8 = (int)(idx % (unsigned)cv) * 8;
  const unsigned p = idx / (unsigned)cv;
  const int bx = (int)(p % (unsigned)w);
  const unsigned prow = p / (unsigned)w;
  const int by = (int)(prow % (unsigned)h);
  const int b = (int)(prow / (unsigned)h);
  const int oy0 = 2 * by, ox0 = 2 * bx;
  int y0[2], x0[2];
  float ly[2], lx[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float fy = (float)(oy0 + r) * ((float)(h - 1) / (float)(oh - 1));
    const float fx = (float)(ox0 + r) * ((float)(w - 1) / (float)(ow - 1));
    y0[r] = (int)fy; x0[r] = (int)fx;
    ly[r] = fy - (float)y0[r]; lx[r] = fx - (float)x0[r];
  }
  const int ldc = split ? 2 * C : C;
  const int dy = y0[1] - y0[0], dx = x0[1] - x0[0];   // 0 or 1 (source step < 0.5), the same for all threads of a block
  if (dy == 0 && dx == 0) upsample_block<0, 0>(in, out, b, h, w, C, split, ldc, c8, oy0, ox0, y0, x0, ly, lx);
  else if (dy == 0) upsample_block<0, 1>(in, out, b, h, w, C, split, ldc, c8, oy0, ox0, y0, x0, ly, lx);
  else if (dx == 0) upsample_block<1, 0>(in, out, b, h, w, C, split, ldc, c8, oy0, ox0, y0, x0, ly, lx);
  else upsample_block<1, 1>(in, out, b, h, w, C, split, ldc, c8, oy0, ox0, y0, x0, ly, lx);
}

// ------------------------------------------------------------------------------------------------
// Pose lift, one thread per ROI.  fp32 steps mirror the torch ops one rounding at a time
// (rot_reps.py:34-55, pose_from_pred_centroid_z.py:74-113); allo->ego in fp64 like the numpy path
// (utils.py:31-88 + transforms3d.axangles.axangle2mat).
__global__ void pose_lift_kernel(const float* __restrict__ raw, int ld, const float* __restrict__ cams,
                                 const float* __restrict__ centers, const float* __restrict__ whs,
                                 const float* __restrict__ ratios, float* __restrict__ out_rot,
                                 float* __restrict__ out_trans, float* __restrict__ out_raw9, int B) {
  ptx::griddep_launch();
  ptx::griddep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const float* r = raw + (long long)i * ld;
  if (out_raw9) {
#pragma unroll
    for (int k = 0; k < 9; ++k) out_raw9[i * 9 + k] = r[k];
  }
  // --- rot6d -> matrix (columns x, y, z) ---
  float a0 = r[0], a1 = r[1], a2 = r[2], b0 = r[3], b1 = r[4], b2 = r[5];
  float na = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(a0, a0), __fmul_rn(a1, a1)), __fmul_rn(a2, a2)));
  na = fmaxf(na, 1e-12f);
  float x0 = __fdiv_rn(a0, na), x1 = __fdiv_rn(a1, na), x2 = __fdiv_rn(a2, na);
  // z = cross(x, y_raw)
  float z0 = __fsub_rn(__fmul_rn(x1, b2), __fmul_rn(x2, b1));
  float z1 = __fsub_rn(__fmul_rn(x2, b0), __fmul_rn(x0, b2));
  float z2 = __fsub_rn(__fmul_rn(x0, b1), __fmul_rn(x1, b0));
  float nz = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(z0, z0), __fmul_rn(z1, z1)), __fmul_rn(z2, z2)));
  nz = fmaxf(nz, 1e-12f);
  z0 = __fdiv_rn(z0, nz); z1 = __fdiv_rn(z1, nz); z2 = __fdiv_rn(z2, nz);
  // y = cross(z, x)
  float y0 = __fsub_rn(__fmul_rn(z1, x2), __fmul_rn(z2, x1));
  float y1 = __fsub_rn(__fmul_rn(z2, x0), __fmul_rn(z0, x2));
  float y2 = __fsub_rn(__fmul_rn(z0, x1), __fmul_rn(z1, x0));
  float Ra[9] = {x0, y0, z0, x1, y1, z1, x2, y2, z2};  // row-major, columns (x,y,z)
  // --- translation ---
  const float* K = cams + i * 9;
  float cx = __fadd_rn(__fmul_rn(r[6], whs[i * 2]), centers[i * 2]);
  float cy = __fadd_rn(__fmul_rn(r[7], whs[i * 2 + 1]), centers[i * 2 + 1]);
  float z = __fmul_rn(r[8], ratios[i]);
  float tx = __fdiv_rn(__fmul_rn(z, __fsub_rn(cx, K[2])), K[0]);
  float ty = __fdiv_rn(__fmul_rn(z, __fsub_rn(cy, K[5])), K[4]);
  out_trans[i * 3] = tx; out_trans[i * 3 + 1] = ty; out_trans[i * 3 + 2] = z;
  // --- allocentric -> egocentric ---
  float nt = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(tx, tx), __fmul_rn(ty, ty)), __fmul_rn(z, z)));
  float ox = __fdiv_rn(tx, nt), oy = __fdiv_rn(ty, nt), oz = __fdiv_rn(z, nt);  // obj_ray (float32)
  double dotv = (double)oz;  // cam_ray (0,0,1) . obj_ray
  double angle = acos(dotv);
  float* Ro = out_rot + i * 9;
  if (angle > 0.0) {
    // axis = cross((0,0,1), obj_ray) = (-oy, ox, 0)
    double ax = -(double)oy, ay = (double)ox, az = 0.0;
    double n = sqrt(ax * ax + ay * ay + az * az);
    ax /= n; ay /= n; az /= n;
    double c = cos(angle), s = sin(angle), Cc = 1.0 - c;
    double xs = ax * s, ys = ay * s, zs = az * s;
    double xC = ax * Cc, yC = ay * Cc, zC = az * Cc;
    double xyC = ax * yC, yzC = ay * zC, zxC = az * xC;
    double M[9] = {ax * xC + c, xyC - zs, zxC + ys, xyC + zs, ay * yC + c, yzC - xs, zxC - ys, yzC + xs, az * zC + c};
#pragma unroll
    for (int rr = 0; rr < 3; ++rr)
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) {
        double acc = M[rr * 3] * (double)Ra[cc] + M[rr * 3 + 1] * (double)Ra[3 + cc] + M[rr * 3 + 2] * (double)Ra[6 + cc];
        Ro[rr * 3 + cc] = (float)acc;
      }
  } else {
#pragma unroll
    for (int k = 0; k < 9; ++k) Ro[k] = Ra[k];
  }
}

}  // namespace

// ================================================================================================
int launch_pack(const float* src, void* dst, int dst_is_bf16, const PackDesc& d, cudaStream_t st) {
  long long total = d.dims[0] * d.dims[1] * d.dims[2] * d.dims[3];
  if (total <= 0) return GDRN_OK;
  long long blocks = (total + 255) / 256;
  if (blocks > 4096) blocks = 4096;
  GDRN_CHECK_CUDA(gdrn_launch_dep(pack_kernel, dim3((int)blocks), dim3(256), 0, st, src, dst, dst_is_bf16, d));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_stem_patchify(const float* img, __nv_bfloat16* out, int B, int H, int W, int split, cudaStream_t st) {
  GDRN_REQUIRE(H % 4 == 0 && W % 4 == 0, "stem: H, W must be multiples of 4");
  long long total = (long long)B * (H / 4) * (W / 4);
  GDRN_CHECK_CUDA(gdrn_launch_dep(stem_patchify_kernel, dim3((int)((total + 127) / 128)), dim3(128), 0, st, img, out, B, H, W, split));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

template <int TW, int TH, int CPC, int R, int MINB>
static int launch_dwconv_cluster(const float* x, const float* w49c, const float* bias, const float* ln_w,
                                 const float* ln_b, __nv_bfloat16* out, int B, int H, int W, int C, float eps,
                                 int split, cudaStream_t st, int c_real) {
  constexpr int IW = TW + 6, IH = TH + 6;
  constexpr int NPIX = TW * TH;
  constexpr int NTHREADS = (CPC / 2) * TH / R;
  const size_t smem = (size_t)(IH * IW * CPC + 49 * CPC + 2 * 8 * (CPC / 64) * NPIX) * sizeof(float) + 32;
  auto kfn = dwconv_ln_cluster_kernel<TW, TH, CPC, R, MINB>;
  GDRN_OPT_IN_SMEM(kfn, smem);
  CUtensorMap tmap;
  {
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[3] = {(uint64_t)C * 4, (uint64_t)W * C * 4, (uint64_t)H * W * C * 4};
    const uint32_t box[4] = {(uint32_t)CPC, (uint32_t)IW, (uint32_t)IH, 1};
    int rc = make_tmap_f32_plain(&tmap, x, 4, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  CUtensorMap tmap_w;
  {
    const uint64_t dims[2] = {(uint64_t)C, 49};
    const uint64_t str[1] = {(uint64_t)C * 4};
    const uint32_t box[2] = {(uint32_t)CPC, 49};
    int rc = make_tmap_f32_plain(&tmap_w, w49c, 2, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(C / CPC, (H / TH) * (W / TW), B);
  cfg.blockDim = dim3(NTHREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = C / CPC;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // see gdrn_launch_dep (common.cuh)
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = gdrn_pdl_enabled() ? 2 : 1;
  static int trace_on = -1;  // GDRN_DW_TRACE=1: phase cycle counts of one mid-grid CTA on stderr (synchronises)
  if (trace_on < 0) trace_on = getenv("GDRN_DW_TRACE") ? 1 : 0;
  static long long* d_trace = nullptr;
  if (trace_on && !d_trace) GDRN_CHECK_CUDA(cudaMalloc(&d_trace, 8 * sizeof(long long)));
  long long* trp = trace_on ? d_trace : nullptr;
  GDRN_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kfn, tmap, tmap_w, bias, ln_w, ln_b, out, B, H, W, C, c_real, eps, split, trp));
  gdrn_count_launch(1);
  if (trace_on) {
    long long h[5];
    GDRN_CHECK_CUDA(cudaMemcpyAsync(h, d_trace, sizeof(h), cudaMemcpyDeviceToHost, st));
    GDRN_CHECK_CUDA(cudaStreamSynchronize(st));
    fprintf(stderr, "[dwconv trace] %dx%d C=%d tile %dx%d R=%d: load-wait=%lld conv=%lld ln-local=%lld cluster-sync=%lld finish=%lld\n",
            H, W, C, TW, TH, R, h[0], h[1], h[2], h[3], h[4]);
  }
  return GDRN_OK;
}

int launch_dwconv_ln(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                     __nv_bfloat16* out, int B, int H, int W, int C, float eps, int split, cudaStream_t st, int c_real) {
  return launch_dwconv_ln_variant(x, w49c, bias, ln_w, ln_b, out, B, H, W, C, eps, split, -1, st, c_real);
}

// variant: -1 = default choice (env GDRN_DW_PP), 0 = one-tile-per-CTA cluster kernel, 1 = persistent ping-pong kernel
int launch_dwconv_ln_variant(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                             __nv_bfloat16* out, int B, int H, int W, int C, float eps, int split, int variant,
                             cudaStream_t st, int c_real) {
  GDRN_REQUIRE(C % 64 == 0 && C <= 1024, "dwconv: C must be a multiple of 64 and <= 1024");
  if (c_real <= 0) c_real = C;
  GDRN_REQUIRE(c_real <= C && C - c_real < 64, "dwconv: c_real must be within the last 64-channel slice of C");
  // cluster kernel: 16x8 tiles x 64 channels (cluster C/64 <= 8) or 8x8 tiles x 128 channels (cluster C/128 <= 8)
  static int rows = -1;  // GDRN_DW_ROWS=2: two output rows per thread (half the LDS traffic, half the warps: measured 4 % slower)
  if (rows < 0) { const char* e = getenv("GDRN_DW_ROWS"); rows = (e && atoi(e) == 2) ? 2 : 1; }
  static int var = -1;   // GDRN_DW_VARIANT: tile-shape experiments
  if (var < 0) { const char* e = getenv("GDRN_DW_VARIANT"); var = e ? atoi(e) : 0; }
#define DW_ARGS x, w49c, bias, ln_w, ln_b, out, B, H, W, C, eps, split, st, c_real
  static int pp = -1;    // GDRN_DW_PP=0: one-tile-per-CTA kernel instead of the persistent ping-pong kernel (A/B experiments)
  if (pp < 0) { const char* e = getenv("GDRN_DW_PP"); pp = e ? atoi(e) : 1; }
  const bool want_pp = variant == 1 || (variant < 0 && pp && var == 0 && rows == 1 && (long long)B * (H / 8) * (W / 16) >= 32);
  if (want_pp) {
    const int rc = launch_dwconv_ln_pp(DW_ARGS);
    if (rc != 1) return rc;
    GDRN_REQUIRE(variant != 1, "dwconv: shape not handled by the ping-pong kernel");
  }
  if (H % 8 == 0 && W % 16 == 0 && C / 64 <= 8) {
    if (var == 1) return launch_dwconv_cluster<16, 4, 64, 1, 3>(DW_ARGS);   // 73 KB: 3 CTAs / SM, 128 threads
    if (var == 2) return launch_dwconv_cluster<8, 8, 64, 1, 3>(DW_ARGS);    // 67 KB: 3 CTAs / SM, 256 threads
    if (var == 3) return launch_dwconv_cluster<8, 4, 64, 1, 4>(DW_ARGS);    // 50 KB: 4 CTAs / SM, 128 threads
    return rows == 2 ? launch_dwconv_cluster<16, 8, 64, 2, 2>(DW_ARGS) : launch_dwconv_cluster<16, 8, 64, 1, 2>(DW_ARGS);
  }
  if (H % 8 == 0 && W % 8 == 0 && C % 128 == 0 && C / 128 <= 8)
    return rows == 2 ? launch_dwconv_cluster<8, 8, 128, 2, 1>(DW_ARGS) : launch_dwconv_cluster<8, 8, 128, 1, 1>(DW_ARGS);
#undef DW_ARGS
  GDRN_REQUIRE(!split, "dwconv: the non-cluster fallback kernel has no split-bf16 output");
  GDRN_REQUIRE(c_real == C && C % 128 == 0, "dwconv: the non-cluster fallback kernel needs C % 128 == 0 and no pad channels");
  const int S = 256 / (C / 4);
  if (W % 16 == 0) {
    long long strips = (long long)B * H * (W / 16);
    GDRN_CHECK_CUDA(gdrn_launch_dep(dwconv_ln_kernel<16>, dim3((int)((strips + S - 1) / S)), dim3(256), 0, st, x, w49c, bias, ln_w, ln_b, out, B, H, W, C, eps));
  } else {
    GDRN_REQUIRE(W % 8 == 0, "dwconv: W must be a multiple of 8");
    long long strips = (long long)B * H * (W / 8);
    GDRN_CHECK_CUDA(gdrn_launch_dep(dwconv_ln_kernel<8>, dim3((int)((strips + S - 1) / S)), dim3(256), 0, st, x, w49c, bias, ln_w, ln_b, out, B, H, W, C, eps));
  }
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_ln_patchify2(const float* x, const float* ln_w, const float* ln_b, __nv_bfloat16* out, int B, int H, int W,
                        int C, float eps, int split, cudaStream_t st, int c_real) {
  GDRN_REQUIRE(C % 64 == 0 && C <= 512 && H % 2 == 0 && W % 2 == 0, "ln_patchify2: unsupported shape");
  if (c_real <= 0) c_real = C;
  GDRN_REQUIRE(c_real <= C, "ln_patchify2: c_real > C");
  const long long total = (long long)B * (H / 2) * (W / 2);
  const int blocks = (int)((total + 7) / 8);
#define LNP_CASE(CC, NV, VW)                                                                                              \
  if (C == CC) {                                                                                                        \
    GDRN_CHECK_CUDA(gdrn_launch_dep(ln_patchify2_kernel<NV, VW>, dim3(blocks), dim3(256), 0, st, x, ln_w, ln_b, out, B, H, W, eps, \
                                    split, c_real));                                                                    \
    gdrn_count_launch(1);                                                                                               \
    return GDRN_OK;                                                                                                     \
  }
  LNP_CASE(128, 1, 4) LNP_CASE(256, 2, 4) LNP_CASE(384, 3, 4) LNP_CASE(512, 4, 4)
  LNP_CASE(64, 1, 2) LNP_CASE(192, 3, 2) LNP_CASE(320, 5, 2) LNP_CASE(448, 7, 2)
#undef LNP_CASE
  GDRN_REQUIRE(false, "ln_patchify2: unsupported channel count");
  return GDRN_ERR_INVALID;
}

int launch_cast_bf16(const float* src, __nv_bfloat16* dst, long long n, cudaStream_t st) {
  long long blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 8192) blocks = 8192;
  GDRN_CHECK_CUDA(gdrn_launch_dep(cast_bf16_kernel, dim3((int)blocks), dim3(256), 0, st, src, dst, n));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_bf16_to_f32(const __nv_bfloat16* src, float* dst, long long n, cudaStream_t st) {
  long long blocks = (n + 255) / 256;
  if (blocks > 8192) blocks = 8192;
  GDRN_CHECK_CUDA(gdrn_launch_dep(bf16_to_f32_kernel, dim3((int)blocks), dim3(256), 0, st, src, dst, n));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_split_to_f32(const __nv_bfloat16* src, float* dst, long long rows, int C, cudaStream_t st) {
  long long blocks = (rows * C + 255) / 256;
  if (blocks > 8192) blocks = 8192;
  GDRN_CHECK_CUDA(gdrn_launch_dep(split_to_f32_kernel, dim3((int)blocks), dim3(256), 0, st, src, dst, rows, C));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_gn_gelu(const void* raw, int raw_is_f32, const double* stats, float* mean_rstd_scratch, const float* gn_w,
                   const float* gn_b, __nv_bfloat16* out, int B, int h, int w, int C, int groups, float eps, int split,
                   cudaStream_t st) {
  GDRN_REQUIRE(C % 8 == 0 && (h * w) % GN_PPT == 0, "gn_gelu: unsupported shape");
  // a 256-thread block covers 256 / (C/8) pixel groups: it must not span more than two images, and 2 * groups <= 256 threads
  GDRN_REQUIRE(groups <= 32 && (long long)(h * w / GN_PPT) * (C / 8) >= 256, "gn_gelu: image too small for the block-level statistics");
  (void)mean_rstd_scratch;
  long long total = (long long)B * (h * w / GN_PPT) * (C / 8);
  GDRN_REQUIRE(total < (1LL << 31), "gn_gelu: tensor too large for 32-bit indexing");
  GDRN_CHECK_CUDA(gdrn_launch_dep(gn_gelu_kernel, dim3((int)((total + 255) / 256)), dim3(256), 0, st, raw, raw_is_f32, stats,
                                  (double)h * w * (C / groups), eps, gn_w, gn_b, out, B, h * w, C, groups, split));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_gn_gelu_f32(const float* raw, const double* stats, float* mean_rstd_scratch, const float* gn_w,
                       const float* gn_b, float* out, int B, int h, int w, int C, int groups, float eps, cudaStream_t st) {
  const int n_bg = B * groups;
  GDRN_CHECK_CUDA(gdrn_launch_dep(gn_finalize_kernel, dim3((n_bg + 127) / 128), dim3(128), 0, st, stats, reinterpret_cast<float2*>(mean_rstd_scratch), n_bg,
                                                        (double)h * w * (C / groups), eps));
  long long total = (long long)B * h * w * C;
  GDRN_CHECK_CUDA(gdrn_launch_dep(gn_gelu_f32_kernel, dim3((int)((total + 255) / 256)), dim3(256), 0, st, raw, reinterpret_cast<const float2*>(mean_rstd_scratch), gn_w,
                                                                gn_b, out, B, h * w, C, groups));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(2);
  return GDRN_OK;
}

int fc_f32_slices(int B, int N, int K) {
  // K slices: enough blocks to cover the chip about twice, slices of whole k tiles, at most FC_MAX_KS
  const int bt = B <= 16 ? 16 : 64;
  const long long blocks = (long long)((N + FC_NB - 1) / FC_NB) * ((B + bt - 1) / bt);
  int ks = 1;
  while (ks < FC_MAX_KS && blocks * ks < 2LL * gdrn_num_sms() && K % (2 * ks * FC_KT) == 0) ks *= 2;
  return ks;
}

size_t fc_f32_part_bytes(int B, int N_max) { return (size_t)FC_MAX_KS * B * N_max * sizeof(float); }

int launch_fc_f32(const float* x, const float* W, const float* bias, float* y, float* part, int B, int N, int K, int ldy, int gelu,
                  cudaStream_t st) {
  GDRN_REQUIRE(K % FC_KT == 0 && N % 4 == 0 && B > 0 && part != nullptr, "fc_f32: K must be a multiple of 32 and N of 4");
  const int ks = fc_f32_slices(B, N, K);
  const int kslice = K / ks;
  if (B <= 16) {
    GDRN_CHECK_CUDA(gdrn_launch_dep(fc_f32_partial_kernel<16>, dim3((N + FC_NB - 1) / FC_NB, ks, (B + 15) / 16), dim3(256), 0, st, x, W,
                                    part, B, N, K, kslice));
  } else {
    GDRN_CHECK_CUDA(gdrn_launch_dep(fc_f32_partial_kernel<64>, dim3((N + FC_NB - 1) / FC_NB, ks, (B + 63) / 64), dim3(256), 0, st, x, W,
                                    part, B, N, K, kslice));
  }
  GDRN_CHECK_CUDA(gdrn_launch_dep(fc_f32_reduce_kernel, dim3((B * (N / 4) + 255) / 256), dim3(256), 0, st, (const float*)part, bias, y, B, N,
                                  ks, ldy, gelu));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(2);
  return GDRN_OK;
}

int launch_cast_split(const float* src, __nv_bfloat16* dst, long long rows, int C, cudaStream_t st) {
  GDRN_REQUIRE(C % 8 == 0, "cast_split: C must be a multiple of 8");
  long long total = rows * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 8192) blocks = 8192;
  GDRN_CHECK_CUDA(gdrn_launch_dep(cast_split_kernel, dim3((int)blocks), dim3(256), 0, st, src, dst, rows, C));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_upsample2x(const __nv_bfloat16* in, __nv_bfloat16* out, int B, int h, int w, int C, int split, cudaStream_t st) {
  GDRN_REQUIRE(C % 8 == 0 && h > 1 && w > 1, "upsample2x: unsupported shape");
  long long total = (long long)B * h * w * (C / 8);   // threads: one per 2 x 2 output block and 8 channels
  GDRN_REQUIRE(total * 4 < (1LL << 31), "upsample2x: tensor too large for 32-bit indexing");
  GDRN_CHECK_CUDA(gdrn_launch_dep(upsample2x_kernel, dim3((int)((total + 255) / 256)), dim3(256), 0, st, in, out, B, h, w, C, split));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

int launch_pose_lift(const float* raw, int ld, const float* cams, const float* centers, const float* whs,
                     const float* ratios, float* out_rot, float* out_trans, float* out_raw9, int B, cudaStream_t st) {
  GDRN_CHECK_CUDA(gdrn_launch_dep(pose_lift_kernel, dim3((B + 63) / 64), dim3(64), 0, st, raw, ld, cams, centers, whs, ratios, out_rot, out_trans, out_raw9, B));
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
