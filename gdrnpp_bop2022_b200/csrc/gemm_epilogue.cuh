// Internal header of the wgmma GEMM kernel (gemm_tc.cu): tile constants, output-row mapping and the epilogues
// (shared-memory accumulator tile or wgmma fragments -> fused math -> global / shared memory).
#pragma once
#include "common.cuh"
#include "gemm_tc.h"

// dynamic shared memory of the GEMM kernel (gemm_tc.cu): accumulator tile, operand ring, epilogue staging, barriers
extern __shared__ uint8_t gemm_smem[];

namespace {

constexpr int BLOCK_M = 128;
constexpr int MMA_K = 16;
constexpr int NUM_THREADS = 384;              // producer warpgroup + 2 MMA / epilogue warpgroups (8 warps)
constexpr int NUM_EPI_WARPS = 8;
constexpr int EPI_STAGE_PITCH = 80;           // 64-byte row segment + 16 B pad (conflict-free 16-byte accesses)
// per epilogue warp: either the TMA-store staging tile (32 rows x 128 B, 128B-swizzled, 1024-aligned), two pairs of
// 16 x 64 B hi / lo tiles (register GELU epilogue) or, for the gather-store path, 32 rows x 80 B + 32 x int64 row map +
// bias/gamma (2 x 128 f32) = 3840 B
constexpr int EPI_STAGE_BYTES = 4096;
constexpr int SMEM_BUDGET = 227 * 1024 - NUM_EPI_WARPS * EPI_STAGE_BYTES - 1024 - 256;

struct RowInfo {
  long long orow;  // output row index
  int b;           // image index (rank 4/5) or row / rows_per_roi
  bool valid;
};

__device__ __forceinline__ RowInfo map_row(const GemmPlan& p, int m_tile, int r) {
  RowInfo ri;
  if (p.a_rank == 2) {
    long long grow = (long long)m_tile * BLOCK_M + r;
    ri.orow = grow;
    ri.valid = grow < p.M;
    ri.b = p.rows_per_roi > 0 ? (int)(grow / p.rows_per_roi) : 0;
  } else {
    int tx = m_tile % p.tiles_x;
    int t2 = m_tile / p.tiles_x;
    int ty = t2 % p.tiles_y;
    int tb = t2 / p.tiles_y;
    int ix = r & ((1 << p.lg_bw) - 1);
    int iy = (r >> p.lg_bw) & ((1 << p.lg_bh) - 1);
    int ib = r >> (p.lg_bw + p.lg_bh);
    int b = (tb << p.lg_bb) + ib;
    int y = (ty << p.lg_bh) + iy;
    int x = (tx << p.lg_bw) + ix;
    ri.b = b;
    ri.valid = b < p.M;
    ri.orow = ((long long)b * p.OH + (y * p.osy + p.ooy)) * p.OW + (x * p.osx + p.oox);
  }
  return ri;
}

template <int CH>
__device__ __forceinline__ void store_row_chunk(const GemmPlan& p, const RowInfo& ri, int col, const float (&v)[CH],
                                                bool f32) {
  // col is a multiple of CH; columns >= N are dropped
  int nvalid = p.N - col;
  if (nvalid <= 0) return;
  if (f32) {
    float* o = reinterpret_cast<float*>(p.out) + ri.orow * p.ldo + col;
    if (nvalid >= CH) {
#pragma unroll
      for (int j = 0; j < CH; j += 4) *reinterpret_cast<float4*>(o + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < CH; ++j)
        if (j < nvalid) o[j] = v[j];
    }
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + ri.orow * p.ldo + col;
    if (nvalid >= CH) {
#pragma unroll
      for (int j = 0; j < CH; j += 8) {
        uint4 u;
        u.x = pack_bf16(v[j], v[j + 1]);
        u.y = pack_bf16(v[j + 2], v[j + 3]);
        u.z = pack_bf16(v[j + 4], v[j + 5]);
        u.w = pack_bf16(v[j + 6], v[j + 7]);
        *reinterpret_cast<uint4*>(o + j) = u;
      }
    } else {
#pragma unroll
      for (int j = 0; j < CH; ++j)
        if (j < nvalid) o[j] = __float2bfloat16(v[j]);
    }
  }
}

template <int CH>
__device__ __forceinline__ void load_vec(const float* __restrict__ src, int col, int N, float (&v)[CH]) {
  if (src == nullptr) {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = 0.f;
    return;
  }
  if (col + CH <= N) {
#pragma unroll
    for (int j = 0; j < CH; j += 4) {
      float4 t = __ldg(reinterpret_cast<const float4*>(src + col + j));
      v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < CH; ++j) v[j] = (col + j < N) ? __ldg(src + col + j) : 0.f;
  }
}

// The accumulator tile lives in shared memory, [BLOCK_M][acc_pitch] fp32 at the 1024-aligned start of the GEMM kernel's
// dynamic shared memory (gemm_tc.cu writes it from the wgmma register fragments).  Epilogues address it as
// (row << 16) | column (the acc_* arguments below); lane l of a warp reads row `row + l`, CH consecutive columns.
// Widths that are multiples of 32 keep dense rows and XOR-swizzle the 16-byte column groups by (row & 7), the others
// pad each row by 16 bytes: either way the 16-byte row reads of 8 consecutive lanes hit distinct banks.
template <int BLOCK_N>
constexpr int acc_pitch() { return BLOCK_N % 32 == 0 ? BLOCK_N : BLOCK_N + 4; }  // floats
template <int BLOCK_N>
constexpr int acc_bytes() { return (BLOCK_M * acc_pitch<BLOCK_N>() * 4 + 1023) / 1024 * 1024; }
template <int BLOCK_N>
__device__ __forceinline__ int acc_index(int row, int col) {  // col: even; a float2 / float4 never straddles groups
  return row * acc_pitch<BLOCK_N>() + (BLOCK_N % 32 == 0 ? col ^ ((row & 7) << 2) : col);
}
__device__ __forceinline__ float* acc_tile() {
  const uint32_t a = ptx::smem_u32(gemm_smem);
  return reinterpret_cast<float*>(gemm_smem + (((a + 1023u) & ~1023u) - a));
}
template <int BLOCK_N, int CH>
__device__ __forceinline__ void acc_load_chunk(uint32_t aaddr, float (&v)[CH]) {
  const float* acc = acc_tile();
  const int row = (aaddr >> 16) + (threadIdx.x & 31), col = aaddr & 0xffff;
#pragma unroll
  for (int j = 0; j < CH; j += 4) {
    const float4 t = *reinterpret_cast<const float4*>(acc + acc_index<BLOCK_N>(row, col + j));
    v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
  }
}

// ------------------------------------------------------------------------------------------------
// Epilogues.  Each of the 128 epilogue threads owns one accumulator row.
// ------------------------------------------------------------------------------------------------
template <int BLOCK_N, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmPlan& p, int m_tile, int n_tile, uint32_t acc_row, int lane,
                                              uint8_t* stg) {
  constexpr int CH = BLOCK_N >= 32 ? 32 : 16;
  const int r = ((threadIdx.x >> 5) & 3) * 32 + lane;
  const RowInfo ri = map_row(p, m_tile, r);
  const int n0 = n_tile * BLOCK_N;

  if constexpr (EPI == EPI_STORE || EPI == EPI_GELU || EPI == EPI_RESID) {
#pragma unroll 1
    for (int c = 0; c < BLOCK_N; c += CH) {
      float v[CH];
      acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
      const int col = n0 + c;
      if (!ri.valid || col >= p.N) continue;
      float bias[CH];
      load_vec<CH>(p.bias, col, p.N, bias);
      if constexpr (EPI == EPI_STORE) {
#pragma unroll
        for (int j = 0; j < CH; ++j) v[j] += bias[j];
        store_row_chunk<CH>(p, ri, col, v, p.out_f32 != 0);
      } else if constexpr (EPI == EPI_GELU) {
#pragma unroll
        for (int j = 0; j < CH; ++j) v[j] = gelu_fast(v[j] + bias[j]);
        store_row_chunk<CH>(p, ri, col, v, false);
      } else {  // EPI_RESID
        float g[CH], x[CH];
        load_vec<CH>(p.gamma, col, p.N, g);
        const float* rs = p.resid + ri.orow * p.ldo + col;
#pragma unroll
        for (int j = 0; j < CH; j += 4) {
          float4 t = *reinterpret_cast<const float4*>(rs + j);
          x[j] = t.x; x[j + 1] = t.y; x[j + 2] = t.z; x[j + 3] = t.w;
        }
#pragma unroll
        for (int j = 0; j < CH; ++j) v[j] = fmaf(g[j], v[j] + bias[j], x[j]);
        store_row_chunk<CH>(p, ri, col, v, true);
      }
    }
  } else if constexpr (EPI == EPI_GNSTATS) {
    const int cpg = p.gn_cpg;  // 4 or 8
#pragma unroll 1
    for (int c = 0; c < BLOCK_N; c += CH) {
      float v[CH];
      acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
      const int col = n0 + c;
      if (col >= p.N) continue;
      if (ri.valid) store_row_chunk<CH>(p, ri, col, v, p.out_f32 != 0);
      // per-group partial sums over this thread's row (stats use the values as stored)
      float s[8], ss[8];
#pragma unroll
      for (int g = 0; g < 8; ++g) { s[g] = 0.f; ss[g] = 0.f; }
      if (!p.out_f32) {
#pragma unroll
        for (int j = 0; j < CH; ++j) v[j] = __bfloat162float(__float2bfloat16(v[j]));
      }
      if (cpg == 8) {
#pragma unroll
        for (int j = 0; j < CH; ++j) { s[j >> 3] += v[j]; ss[j >> 3] = fmaf(v[j], v[j], ss[j >> 3]); }
      } else {
#pragma unroll
        for (int j = 0; j < CH; ++j) { s[j >> 2] += v[j]; ss[j >> 2] = fmaf(v[j], v[j], ss[j >> 2]); }
      }
      const int ng = CH / cpg;  // groups in this chunk (4 or 8)
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        if (g < ng) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            s[g] += __shfl_xor_sync(0xffffffffu, s[g], o);
            ss[g] += __shfl_xor_sync(0xffffffffu, ss[g], o);
          }
        }
      }
      if (ri.valid) {  // warp-uniform: a warp's 32 rows lie in one image
        double* st = p.gn_stats + ((long long)ri.b * p.gn_groups + col / cpg) * 2;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          if (g < ng && lane == g) {
            atomicAdd(st + 2 * g, (double)s[g]);
            atomicAdd(st + 2 * g + 1, (double)ss[g]);
          }
        }
      }
    }
  } else if constexpr (EPI == EPI_BIAS_LN) {
    // N <= BLOCK_N (N % 32 == 0): the thread sees the whole channel vector of its pixel. Three passes over the accumulator row.
    float sum = 0.f;
#pragma unroll 1
    for (int c = 0; c < p.N; c += CH) {
      float v[CH], bias[CH];
      acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
      load_vec<CH>(p.bias, c, p.N, bias);
#pragma unroll
      for (int j = 0; j < CH; ++j) sum += v[j] + bias[j];
    }
    const int ln_n = p.ln_n > 0 ? p.ln_n : p.N;
    const float mean = sum / (float)ln_n;
    // centred sum of squares over the ln_n real columns only: the zero pad columns are masked out of the pass (subtracting
    // their (N - ln_n) * mean^2 afterwards cancels catastrophically when |mean| >> std)
    float sq = 0.f;
#pragma unroll 1
    for (int c = 0; c < p.N; c += CH) {
      float v[CH], bias[CH];
      acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
      load_vec<CH>(p.bias, c, p.N, bias);
#pragma unroll
      for (int j = 0; j < CH; ++j) { const float d = c + j < ln_n ? v[j] + bias[j] - mean : 0.f; sq = fmaf(d, d, sq); }
    }
    const float rstd = rsqrtf(sq / (float)ln_n + p.ln_eps);
#pragma unroll 1
    for (int c = 0; c < p.N; c += CH) {
      float v[CH], bias[CH], w[CH], bb[CH];
      acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
      load_vec<CH>(p.bias, c, p.N, bias);
      load_vec<CH>(p.ln_w, c, p.N, w);
      load_vec<CH>(p.ln_b, c, p.N, bb);
#pragma unroll
      for (int j = 0; j < CH; ++j) v[j] = fmaf((v[j] + bias[j] - mean) * rstd, w[j], bb[j]);
      if constexpr (CH == 32) {
        if (p.use_tma_store) {  // 32 rows x 128 B staging tile (SWIZZLE_128B) -> one TMA store, rows >= M clipped
          if (lane == 0) ptx::bulk_wait_read0();
          __syncwarp();
          uint4* dst = reinterpret_cast<uint4*>(stg + lane * 128);
          const int sw = lane & 7;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            dst[j ^ sw] = make_uint4(__float_as_uint(v[4 * j]), __float_as_uint(v[4 * j + 1]), __float_as_uint(v[4 * j + 2]),
                                     __float_as_uint(v[4 * j + 3]));
          ptx::fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            ptx::tma_store_2d(&p.tmap_out, ptx::smem_u32(stg), c, m_tile * BLOCK_M + (int)((threadIdx.x >> 5) & 3) * 32);
            ptx::bulk_commit();
          }
          continue;
        }
      }
      if (ri.valid) store_row_chunk<CH>(p, ri, c, v, true);
    }
  } else if constexpr (EPI == EPI_OUTCONV) {
    // BLOCK_N == 80: [vis, full, x, y, z, region_0..64, pad x10] of the ROI's own class
    // (GDRN_double_mask.py:107-126 gather + :131-148 feature assembly + conv_pnp_net.py:130-136).
    float v[80];
    {
      float t[32];
      acc_load_chunk<BLOCK_N, 32>(acc_row, t);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = t[j];
      acc_load_chunk<BLOCK_N, 32>(acc_row + 32, t);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[32 + j] = t[j];
      float t16[16];
      acc_load_chunk<BLOCK_N, 16>(acc_row + 64, t16);
#pragma unroll
      for (int j = 0; j < 16; ++j) v[64 + j] = t16[j];
    }
    if (ri.valid) {
      const int b = ri.b;
      const int pix = (int)(ri.orow - (long long)b * p.rows_per_roi);
      int cls = p.roi_classes ? (int)p.roi_classes[b] : 0;
      cls = cls < 0 ? 0 : (cls >= p.num_classes ? p.num_classes - 1 : cls);
      const float* ob = p.oc_bias + cls * 80;
#pragma unroll
      for (int j = 0; j < 72; j += 4) {
        float4 t = __ldg(reinterpret_cast<const float4*>(ob + j));
        v[j] += t.x; v[j + 1] += t.y; v[j + 2] += t.z; v[j + 3] += t.w;
      }
      const long long hw = p.rows_per_roi;
      if (p.map_mask) {
        p.map_mask[(long long)b * hw + pix] = v[0];
        p.map_full[(long long)b * hw + pix] = v[1];
        p.map_x[(long long)b * hw + pix] = v[2];
        p.map_y[(long long)b * hw + pix] = v[3];
        p.map_z[(long long)b * hw + pix] = v[4];
#pragma unroll
        for (int j = 0; j < 65; ++j) p.map_region[((long long)b * 65 + j) * hw + pix] = v[5 + j];
      }
      // softmax over region[1:65] = v[6..69]
      float mx = v[6];
#pragma unroll
      for (int j = 7; j < 70; ++j) mx = fmaxf(mx, v[j]);
      float den = 0.f;
#pragma unroll
      if (p.split) {  // precise mode: full-accuracy exp
#pragma unroll
        for (int j = 6; j < 70; ++j) { v[j] = expf(v[j] - mx); den += v[j]; }
      } else {
#pragma unroll
        for (int j = 6; j < 70; ++j) { v[j] = __expf(v[j] - mx); den += v[j]; }
      }
      const float inv = 1.0f / den;
      const float ex = __ldg(p.roi_extents + b * 3 + 0), ey = __ldg(p.roi_extents + b * 3 + 1),
                  ez = __ldg(p.roi_extents + b * 3 + 2);
      float f[72];
      f[0] = (v[2] - 0.5f) * ex;
      f[1] = (v[3] - 0.5f) * ey;
      f[2] = (v[4] - 0.5f) * ez;
      f[3] = __ldg(p.roi_coord_2d + ((long long)b * 2 + 0) * hw + pix);
      f[4] = __ldg(p.roi_coord_2d + ((long long)b * 2 + 1) * hw + pix);
#pragma unroll
      for (int j = 0; j < 64; ++j) f[5 + j] = v[6 + j] * inv;
      f[69] = 0.f; f[70] = 0.f; f[71] = 0.f;
      const int pw = p.split ? 256 : 128;  // Patch-PnP input row width (split mode: [hi 128 | lo 128])
      uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.pnp_in) + ri.orow * pw);
#pragma unroll
      for (int j = 0; j < 72; j += 8) {
        uint4 u;
        u.x = pack_bf16(f[j], f[j + 1]);
        u.y = pack_bf16(f[j + 2], f[j + 3]);
        u.z = pack_bf16(f[j + 4], f[j + 5]);
        u.w = pack_bf16(f[j + 6], f[j + 7]);
        dst[j >> 3] = u;
      }
#pragma unroll
      for (int j = 9; j < 16; ++j) dst[j] = make_uint4(0, 0, 0, 0);
      if (p.split) {
#pragma unroll
        for (int j = 0; j < 72; ++j) f[j] = f[j] - __bfloat162float(__float2bfloat16(f[j]));
#pragma unroll
        for (int j = 0; j < 72; j += 8) {
          uint4 u;
          u.x = pack_bf16(f[j], f[j + 1]);
          u.y = pack_bf16(f[j + 2], f[j + 3]);
          u.z = pack_bf16(f[j + 4], f[j + 5]);
          u.w = pack_bf16(f[j + 6], f[j + 7]);
          dst[16 + (j >> 3)] = u;
        }
#pragma unroll
        for (int j = 25; j < 32; ++j) dst[j] = make_uint4(0, 0, 0, 0);
      }
    }
  }
}


// GELU mode 2: fp32 tanh form with the hardware tanh.approx.f32 (1 MUFU / element):
// 0.5*x*(1 + tanh(x*(c0 + c1*x^2 + c2*x^4))) with (c0,c1,c2) fitted to the erf form (tools/fit_gelu.py).
__device__ __forceinline__ float gelu_tanh_f32(float x) {
  const float xc = fminf(fmaxf(x, -8.f), 8.f);  // the fitted polynomial changes sign beyond |x| ~ 11
  const float x2 = xc * xc;
  float p = fmaf(x2, GELU_T2, GELU_T1);
  p = fmaf(p, x2, GELU_T0);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(xc * p));
  const float hx = 0.5f * x;
  return fmaf(hx, t, hx);
}

// Epilogue for EPI_STORE / EPI_GELU / EPI_RESID / EPI_GNSTATS with coalesced global traffic.
// Eight warps: warp ew owns accumulator rows [32*(ew&3), +32) and the column half (ew>>2) of the tile.  A thread owns
// one accumulator row; 64-byte row segments (32 bf16 or 16 fp32 columns) are staged in the warp's private
// shared-memory buffer (pitch 80 B, conflict-free 16-byte accesses) and then written (and, for the residual,
// first read) with 16-byte accesses in which 4 lanes cover one row segment: every warp-wide access touches
// eight full 64-byte runs (16 whole sectors) instead of 32 scattered 16-byte pieces.
template <int BLOCK_N, int EPI, bool F32>
__device__ __forceinline__ void epilogue_tile_staged_t(const GemmPlan& p, int m_tile, int n_tile, uint32_t acc_base,
                                                       int ew, int lane, uint8_t* stg) {
  static_assert(BLOCK_N >= 64, "staged epilogue needs BLOCK_N >= 64");
  constexpr int CPW = BLOCK_N / 2;      // columns per warp
  constexpr int CH = F32 ? 16 : 32;     // columns per staged row segment (64 bytes)
  constexpr int ESZ = F32 ? 4 : 2;
  const int q = ew & 3, half = ew >> 2;
  const int r = q * 32 + lane;
  const RowInfo ri = map_row(p, m_tile, r);
  long long* s_orow = reinterpret_cast<long long*>(stg + 32 * EPI_STAGE_PITCH);
  const float* s_bias = reinterpret_cast<const float*>(stg + 32 * EPI_STAGE_PITCH + 256);  // [128] bias, [128] gamma
  s_orow[lane] = ri.valid ? ri.orow : -1;
  __syncwarp();
  const int n0 = n_tile * BLOCK_N + half * CPW;
  const uint32_t acc_row = acc_base + ((uint32_t)(q * 32) << 16) + half * CPW;
  uint8_t* my_row = stg + lane * EPI_STAGE_PITCH;
  const int cpg = p.gn_cpg;
  const int fl_row = lane >> 2, fl_piece = lane & 3;  // flush / prefetch mapping: 8 rows x 4 pieces per pass
  uint4 rres[4];
  if constexpr (EPI == EPI_RESID) {
    if (n0 < p.N) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const long long orow = s_orow[k * 8 + fl_row];
        rres[k] = (orow >= 0) ? *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.resid + orow * p.ldo + n0) + fl_piece * 16)
                              : make_uint4(0, 0, 0, 0);
      }
    }
  }

#pragma unroll 1
  for (int c = 0; c < CPW; c += CH) {
    const int col = n0 + c;
    if (col >= p.N) break;  // warp-uniform
    if constexpr (EPI == EPI_RESID) {
      // residual segment rows: registers (fetched one chunk ahead, see below) -> staging buffer
#pragma unroll
      for (int k = 0; k < 4; ++k) *reinterpret_cast<uint4*>(stg + (k * 8 + fl_row) * EPI_STAGE_PITCH + fl_piece * 16) = rres[k];
      // issue the coalesced loads of the NEXT chunk now; they complete while this chunk is processed
      if (c + CH < CPW && col + CH < p.N) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const long long orow = s_orow[k * 8 + fl_row];
          rres[k] = (orow >= 0) ? *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.resid + orow * p.ldo + col + CH) + fl_piece * 16)
                                : make_uint4(0, 0, 0, 0);
        }
      }
      __syncwarp();
    }
    float v[CH];
    acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
    if constexpr (EPI == EPI_STORE || EPI == EPI_GELU) {
      const float4* sb = reinterpret_cast<const float4*>(s_bias + c);  // warp-wide broadcast reads
#pragma unroll
      for (int j = 0; j < CH; j += 4) {
        const float4 b4 = sb[j >> 2];
        v[j] += b4.x; v[j + 1] += b4.y; v[j + 2] += b4.z; v[j + 3] += b4.w;
      }
    } else if constexpr (EPI == EPI_RESID) {
      float bias[CH], g[CH];
      {
        const float4* sb = reinterpret_cast<const float4*>(s_bias + c);
        const float4* sg = reinterpret_cast<const float4*>(s_bias + 128 + c);
#pragma unroll
        for (int j = 0; j < CH; j += 4) {
          const float4 b4 = sb[j >> 2], g4 = sg[j >> 2];
          bias[j] = b4.x; bias[j + 1] = b4.y; bias[j + 2] = b4.z; bias[j + 3] = b4.w;
          g[j] = g4.x; g[j + 1] = g4.y; g[j + 2] = g4.z; g[j + 3] = g4.w;
        }
      }
      const float4* xr = reinterpret_cast<const float4*>(my_row);
#pragma unroll
      for (int j = 0; j < CH; j += 4) {
        const float4 x = xr[j >> 2];
        v[j] = fmaf(g[j], v[j] + bias[j], x.x);
        v[j + 1] = fmaf(g[j + 1], v[j + 1] + bias[j + 1], x.y);
        v[j + 2] = fmaf(g[j + 2], v[j + 2] + bias[j + 2], x.z);
        v[j + 3] = fmaf(g[j + 3], v[j + 3] + bias[j + 3], x.w);
      }
    }
    // ---- registers -> staging row ----
    if constexpr (F32) {
      float4* dst = reinterpret_cast<float4*>(my_row);
#pragma unroll
      for (int j = 0; j < CH; j += 4) dst[j >> 2] = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    } else {
      uint4* dst = reinterpret_cast<uint4*>(my_row);
      if (EPI == EPI_GELU && p.gelu_mode == 1) {
#pragma unroll
        for (int j = 0; j < CH; j += 8) {
          uint4 w;
          w.x = gelu_pack2_f16(v[j], v[j + 1]); w.y = gelu_pack2_f16(v[j + 2], v[j + 3]);
          w.z = gelu_pack2_f16(v[j + 4], v[j + 5]); w.w = gelu_pack2_f16(v[j + 6], v[j + 7]);
          dst[j >> 3] = w;
        }
      } else {
        if constexpr (EPI == EPI_GELU) {
          if (p.gelu_mode == 3) {
#pragma unroll
            for (int j = 0; j < CH; ++j) v[j] = gelu_erf(v[j]);
          } else if (p.gelu_mode == 2) {
#pragma unroll
            for (int j = 0; j < CH; ++j) v[j] = gelu_tanh_f32(v[j]);
          } else {
#pragma unroll
            for (int j = 0; j < CH; ++j) v[j] = gelu_fast(v[j]);
          }
        }
#pragma unroll
        for (int j = 0; j < CH; j += 8) {
          uint4 w;
          w.x = pack_bf16(v[j], v[j + 1]); w.y = pack_bf16(v[j + 2], v[j + 3]);
          w.z = pack_bf16(v[j + 4], v[j + 5]); w.w = pack_bf16(v[j + 6], v[j + 7]);
          dst[j >> 3] = w;
        }
      }
    }
    if constexpr (EPI == EPI_GNSTATS) {
      // per-(image, group) sum / sum of squares of the values as stored
      constexpr int NG_MAX = CH / 4;
      float s[NG_MAX], ss[NG_MAX];
#pragma unroll
      for (int g = 0; g < NG_MAX; ++g) { s[g] = 0.f; ss[g] = 0.f; }
      if (!F32) {
#pragma unroll
        for (int j = 0; j < CH; ++j) v[j] = __bfloat162float(__float2bfloat16(v[j]));
      }
      if (cpg == 8) {
#pragma unroll
        for (int j = 0; j < CH; ++j) { s[j >> 3] += v[j]; ss[j >> 3] = fmaf(v[j], v[j], ss[j >> 3]); }
      } else {
#pragma unroll
        for (int j = 0; j < CH; ++j) { s[j >> 2] += v[j]; ss[j >> 2] = fmaf(v[j], v[j], ss[j >> 2]); }
      }
      const int ng = CH / cpg;
#pragma unroll
      for (int g = 0; g < NG_MAX; ++g) {
        if (g < ng) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            s[g] += __shfl_xor_sync(0xffffffffu, s[g], o);
            ss[g] += __shfl_xor_sync(0xffffffffu, ss[g], o);
          }
        }
      }
      if (ri.valid) {  // warp-uniform: a warp's 32 rows lie in one image
        double* st = p.gn_stats + ((long long)ri.b * p.gn_groups + col / cpg) * 2;
#pragma unroll
        for (int g = 0; g < NG_MAX; ++g) {
          if (g < ng && lane == g) {
            atomicAdd(st + 2 * g, (double)s[g]);
            atomicAdd(st + 2 * g + 1, (double)ss[g]);
          }
        }
      }
    }
    __syncwarp();
    // ---- coalesced flush of the 32 row segments ----
#pragma unroll
    for (int pass = 0; pass < 32; pass += 8) {
      const int rr = pass + fl_row;
      const long long orow = s_orow[rr];
      if (orow >= 0)
        *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(p.out) + (orow * p.ldo + col) * ESZ + fl_piece * 16) =
            *reinterpret_cast<const uint4*>(stg + rr * EPI_STAGE_PITCH + fl_piece * 16);
    }
    __syncwarp();
  }
}


// Epilogue for rank-2 outputs (EPI_STORE / EPI_GELU / EPI_RESID) with TMA stores.
// Eight warps as above.  A thread owns one accumulator row; it writes 128-byte row segments (64 bf16 or 32 fp32
// columns, produced as two 64-byte halves) into the warp's 32 x 128 B staging tile in the
// SWIZZLE_128B layout (16-byte piece j of row r at piece j ^ (r & 7): conflict-free row-wise STS.128), and one lane
// issues a single cp.async.bulk.tensor store per tile.  No address arithmetic, LDS or STG in the flush; rows beyond
// M are clipped by the tensor map.  The residual of EPI_RESID is read by its owner thread (64 contiguous bytes per
// half, register-prefetched one half ahead).
template <int BLOCK_N, int EPI, bool F32>
__device__ __forceinline__ void epilogue_tile_tma(const GemmPlan& p, int m_tile, int n_tile, uint32_t acc_base, int ew,
                                                  int lane, uint8_t* stg) {
  static_assert(BLOCK_N >= 128, "TMA-store epilogue needs BLOCK_N >= 128");
  constexpr int CPW = BLOCK_N / 2;      // columns per warp
  constexpr int CH = F32 ? 16 : 32;     // columns per 64-byte half row
  constexpr int GW = 2 * CH;            // columns per staged 128-byte row (one TMA store)
  const int q = ew & 3, half = ew >> 2;
  const long long grow = (long long)m_tile * BLOCK_M + q * 32 + lane;
  const bool rvalid = grow < p.M;
  const int n0 = n_tile * BLOCK_N + half * CPW;
  const uint32_t acc_row = acc_base + ((uint32_t)(q * 32) << 16) + half * CPW;
  const uint32_t stg_u32 = ptx::smem_u32(stg);
  uint8_t* my_row = stg + lane * 128;
  const int sw = lane & 7;

  uint4 rres[4];
  const float* rrow = nullptr;
  const bool red = (EPI == EPI_RESID) && p.resid_reduce;  // launch-uniform: out += gamma*(acc+bias) by TMA reduce-add
  if constexpr (EPI == EPI_RESID) {
    rrow = p.resid + grow * p.ldo + n0;
    if (rvalid && n0 < p.N && !red) {
#pragma unroll
      for (int k = 0; k < 4; ++k) rres[k] = *reinterpret_cast<const uint4*>(rrow + 4 * k);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) rres[k] = make_uint4(0, 0, 0, 0);
    }
  }

#pragma unroll 1
  for (int g = 0; g < CPW; g += GW) {
    const int gcol = n0 + g;
    if (gcol >= p.N) break;  // warp-uniform
    // the previous store of this warp must have finished reading the staging tile
    if (lane == 0) ptx::bulk_wait_read0();
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = g + h * CH;
      const int col = n0 + c;
      // bias is read four columns at a time right where it is consumed (keeps the live register set small); the loads
      // are warp-uniform L1 hits
      auto bias4 = [&](int j) {
        return p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + col + j)) : make_float4(0.f, 0.f, 0.f, 0.f);
      };
      float x[EPI == EPI_RESID ? CH : 1], gm[EPI == EPI_RESID ? CH : 1];
      if constexpr (EPI == EPI_RESID) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          x[4 * k] = __uint_as_float(rres[k].x); x[4 * k + 1] = __uint_as_float(rres[k].y);
          x[4 * k + 2] = __uint_as_float(rres[k].z); x[4 * k + 3] = __uint_as_float(rres[k].w);
          const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.gamma + col + 4 * k));
          gm[4 * k] = g4.x; gm[4 * k + 1] = g4.y; gm[4 * k + 2] = g4.z; gm[4 * k + 3] = g4.w;
        }
        // next half's residual: in flight while this half is processed
        if (rvalid && !red && c + CH < CPW && col + CH < p.N) {
#pragma unroll
          for (int k = 0; k < 4; ++k) rres[k] = *reinterpret_cast<const uint4*>(rrow + c + CH + 4 * k);
        }
      }
      float v[CH];
      acc_load_chunk<BLOCK_N, CH>(acc_row + c, v);
      uint4* dst = reinterpret_cast<uint4*>(my_row);
      if constexpr (F32) {
        if constexpr (EPI == EPI_RESID) {
#pragma unroll
          for (int j = 0; j < CH; j += 4) {
            const float4 b4 = bias4(j);
            v[j] = fmaf(gm[j], v[j] + b4.x, x[j]); v[j + 1] = fmaf(gm[j + 1], v[j + 1] + b4.y, x[j + 1]);
            v[j + 2] = fmaf(gm[j + 2], v[j + 2] + b4.z, x[j + 2]); v[j + 3] = fmaf(gm[j + 3], v[j + 3] + b4.w, x[j + 3]);
          }
        } else {
#pragma unroll
          for (int j = 0; j < CH; j += 4) {
            const float4 b4 = bias4(j);
            v[j] += b4.x; v[j + 1] += b4.y; v[j + 2] += b4.z; v[j + 3] += b4.w;
          }
        }
#pragma unroll
        for (int j = 0; j < CH; j += 4)
          dst[(h * 4 + (j >> 2)) ^ sw] = make_uint4(__float_as_uint(v[j]), __float_as_uint(v[j + 1]),
                                                    __float_as_uint(v[j + 2]), __float_as_uint(v[j + 3]));
      } else {
        if (EPI == EPI_GELU && p.gelu_mode == 1) {
#pragma unroll
          for (int j = 0; j < CH; j += 8) {
            const float4 ba = bias4(j), bb = bias4(j + 4);
            v[j] += ba.x; v[j + 1] += ba.y; v[j + 2] += ba.z; v[j + 3] += ba.w;
            v[j + 4] += bb.x; v[j + 5] += bb.y; v[j + 6] += bb.z; v[j + 7] += bb.w;
            uint4 w;
            w.x = gelu_pack2_f16(v[j], v[j + 1]); w.y = gelu_pack2_f16(v[j + 2], v[j + 3]);
            w.z = gelu_pack2_f16(v[j + 4], v[j + 5]); w.w = gelu_pack2_f16(v[j + 6], v[j + 7]);
            dst[(h * 4 + (j >> 3)) ^ sw] = w;
          }
        } else {
#pragma unroll
          for (int j = 0; j < CH; j += 4) {
            const float4 b4 = bias4(j);
            v[j] += b4.x; v[j + 1] += b4.y; v[j + 2] += b4.z; v[j + 3] += b4.w;
          }
          if constexpr (EPI == EPI_GELU) {
            if (p.gelu_mode == 3) {
#pragma unroll
              for (int j = 0; j < CH; ++j) v[j] = gelu_erf(v[j]);
            } else if (p.gelu_mode == 2) {
#pragma unroll
              for (int j = 0; j < CH; ++j) v[j] = gelu_tanh_f32(v[j]);
            } else {
#pragma unroll
              for (int j = 0; j < CH; ++j) v[j] = gelu_fast(v[j]);
            }
          }
#pragma unroll
          for (int j = 0; j < CH; j += 8) {
            uint4 w;
            w.x = pack_bf16(v[j], v[j + 1]); w.y = pack_bf16(v[j + 2], v[j + 3]);
            w.z = pack_bf16(v[j + 4], v[j + 5]); w.w = pack_bf16(v[j + 6], v[j + 7]);
            dst[(h * 4 + (j >> 3)) ^ sw] = w;
          }
        }
      }
    }
    ptx::fence_proxy_async();  // generic-proxy smem writes -> visible to the TMA (async proxy)
    __syncwarp();
    if (lane == 0) {
      if (red) ptx::tma_reduce_add_2d(&p.tmap_out, stg_u32, gcol, m_tile * BLOCK_M + q * 32);
      else ptx::tma_store_2d(&p.tmap_out, stg_u32, gcol, m_tile * BLOCK_M + q * 32);
      ptx::bulk_commit();
    }
  }
}

// Epilogues straight from the wgmma accumulator fragments: split-bf16 rank-2 GEMMs with EPI_STORE (fp32 out), EPI_GELU
// ([hi N | lo N] bf16 out) and EPI_RESID, i.e. the ConvNeXt MLPs and downsamples (gemm_tc_launch picks them).  Warp wl of
// consumer warpgroup wg holds tile rows w = 64 wg + 16 wl + (lane >> 2) and w + 8 (`wrow` = 64 wg + 16 wl) and, of every
// 8-column group j, the columns 8 j + 2 (lane & 3) + {0, 1}: acc[4 j], acc[4 j + 1] on row w, acc[4 j + 2], acc[4 j + 3] on
// row w + 8.  The arithmetic per element is that of the accumulator-tile epilogues, operation for operation.
// Rows >= M and columns >= N are neither read nor written.

// EPI_RESID: this thread's residual pairs x[2 j + h] (row w + 8 h, group j), loaded before the last MMAs retire
template <int BLOCK_N>
__device__ __forceinline__ void frag_resid_load(const GemmPlan& p, int m_tile, int n_tile, int wrow, int lane,
                                                float2 (&x)[BLOCK_N / 4]) {
  const long long r0 = (long long)m_tile * BLOCK_M + wrow + (lane >> 2);
  const int c0 = n_tile * BLOCK_N + (lane & 3) * 2;
  // two row pointers and immediate column offsets: no per-element address registers next to the accumulators
  const float* xr[2] = {p.resid + r0 * p.ldo + c0, p.resid + (r0 + 8) * p.ldo + c0};
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      x[2 * j + h] = (r0 + 8 * h < p.M && c0 + 8 * j < p.N) ? *reinterpret_cast<const float2*>(xr[h] + 8 * j) : make_float2(0.f, 0.f);
  }
}

// EPI_GELU: per 32-column chunk, bias + exact-erf GELU + hi / lo split as element pairs, then hi and lo go into two
// 16-row x 64-byte tiles of the warp's staging slot (SWIZZLE_64B: 16-byte piece c of row r at c ^ ((r >> 1) & 3), so the
// 4-byte stores of a warp hit 32 distinct banks) and one lane issues two TMA stores (map box {32, 16}): hi at column
// `col`, lo at N + col; the map clips rows >= M.  The slot holds two such pairs, used in turn (`sbuf` counts the chunks
// this warp has stored), so a chunk's stores may still be reading while the next chunk is written.
template <int BLOCK_N, int EPI>
__device__ __forceinline__ void epilogue_regs(const GemmPlan& p, int m_tile, int n_tile, int wrow, int lane,
                                              const float (&acc)[BLOCK_N / 2], const float2 (&x)[EPI == EPI_RESID ? BLOCK_N / 4 : 1],
                                              uint8_t* stg, uint32_t& sbuf) {
  static_assert(EPI == EPI_STORE || EPI == EPI_GELU || EPI == EPI_RESID, "register epilogue: STORE / GELU / RESID only");
  const long long r0 = (long long)m_tile * BLOCK_M + wrow + (lane >> 2);
  const int c0 = n_tile * BLOCK_N + (lane & 3) * 2;
  if constexpr (EPI == EPI_GELU) {
    const int sw = (lane >> 3) & 3;   // ((lane >> 2) >> 1) & 3; the same for row + 8
#pragma unroll
    for (int ch = 0; ch < BLOCK_N / 32; ++ch) {
      const int col = n_tile * BLOCK_N + ch * 32;
      if (col >= p.N) break;   // warp-uniform
      f32x2_t v2[8];           // [2 jj + h]: group 4 ch + jj, row w + 8 h
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) v2[2 * jj + h] = f2_pack(acc[4 * (4 * ch + jj) + 2 * h], acc[4 * (4 * ch + jj) + 2 * h + 1]);
      }
      if (p.bias) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + c0 + ch * 32 + 8 * jj));
          v2[2 * jj] = f2_add(v2[2 * jj], f2_pack(b.x, b.y));
          v2[2 * jj + 1] = f2_add(v2[2 * jj + 1], f2_pack(b.x, b.y));
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) v2[j] = gelu_erf2(v2[j]);
      uint32_t hi[8], lo[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 f = f2_unpack(v2[j]);
        const uint32_t hb = pack_bf16(f.x, f.y);
        hi[j] = hb;
        const float2 d = f2_unpack(f2_sub(v2[j], f2_pack(__uint_as_float(hb << 16), __uint_as_float(hb & 0xffff0000u))));
        lo[j] = pack_bf16(d.x, d.y);
      }
      if (lane == 0) ptx::bulk_wait_read1();   // the stores issued from this half of the slot two chunks ago have read it
      __syncwarp();
      uint8_t* buf = stg + (sbuf & 1u) * 2048u;   // [hi 16 x 64 B | lo 16 x 64 B]
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int off = ((lane >> 2) + 8 * h) * 64 + ((jj ^ sw) << 4) + (lane & 3) * 4;
          *reinterpret_cast<uint32_t*>(buf + off) = hi[2 * jj + h];
          *reinterpret_cast<uint32_t*>(buf + 1024 + off) = lo[2 * jj + h];
        }
      }
      ptx::fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        const uint32_t src = ptx::smem_u32(buf);
        const int row0 = m_tile * BLOCK_M + wrow;
        ptx::tma_store_2d(&p.tmap_out, src, col, row0);
        ptx::tma_store_2d(&p.tmap_out, src + 1024, p.N + col, row0);
        ptx::bulk_commit();
      }
      ++sbuf;
    }
  } else {
    // fp32 out: 8-byte stores, four lanes fill one 32-byte sector of a row
    float* orow[2] = {reinterpret_cast<float*>(p.out) + r0 * p.ldo + c0, reinterpret_cast<float*>(p.out) + (r0 + 8) * p.ldo + c0};
    const bool rv[2] = {r0 < p.M, r0 + 8 < p.M};
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int c = c0 + 8 * j;
      if (c >= p.N) continue;
      const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + c)) : make_float2(0.f, 0.f);
      const float2 g = EPI == EPI_RESID ? __ldg(reinterpret_cast<const float2*>(p.gamma + c)) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!rv[h]) continue;
        float2 v = make_float2(acc[4 * j + 2 * h] + b.x, acc[4 * j + 2 * h + 1] + b.y);
        if constexpr (EPI == EPI_RESID) v = make_float2(fmaf(g.x, v.x, x[2 * j + h].x), fmaf(g.y, v.y, x[2 * j + h].y));
        *reinterpret_cast<float2*>(orow[h] + 8 * j) = v;
      }
    }
  }
}

template <int BLOCK_N, int EPI>
__device__ __forceinline__ void epilogue_tile_staged(const GemmPlan& p, int m_tile, int n_tile, uint32_t acc_base,
                                                     int ew, int lane, uint8_t* stg) {
  if constexpr (BLOCK_N >= 128 && (EPI == EPI_STORE || EPI == EPI_GELU || EPI == EPI_RESID)) {
    if (p.use_tma_store) {  // launch-uniform
      if constexpr (EPI == EPI_RESID) {
        epilogue_tile_tma<BLOCK_N, EPI, true>(p, m_tile, n_tile, acc_base, ew, lane, stg);
      } else if constexpr (EPI == EPI_GELU) {
        epilogue_tile_tma<BLOCK_N, EPI, false>(p, m_tile, n_tile, acc_base, ew, lane, stg);
      } else {
        if (p.out_f32) epilogue_tile_tma<BLOCK_N, EPI, true>(p, m_tile, n_tile, acc_base, ew, lane, stg);
        else epilogue_tile_tma<BLOCK_N, EPI, false>(p, m_tile, n_tile, acc_base, ew, lane, stg);
      }
      return;
    }
  }
  if constexpr (EPI == EPI_RESID) {
    epilogue_tile_staged_t<BLOCK_N, EPI, true>(p, m_tile, n_tile, acc_base, ew, lane, stg);
  } else if constexpr (EPI == EPI_GELU) {
    epilogue_tile_staged_t<BLOCK_N, EPI, false>(p, m_tile, n_tile, acc_base, ew, lane, stg);
  } else {
    if (p.out_f32) epilogue_tile_staged_t<BLOCK_N, EPI, true>(p, m_tile, n_tile, acc_base, ew, lane, stg);
    else epilogue_tile_staged_t<BLOCK_N, EPI, false>(p, m_tile, n_tile, acc_base, ew, lane, stg);
  }
}

}  // namespace
