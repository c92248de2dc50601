// Fused ConvNeXt MLP block (stage 0, C = 128): x += gamma * (W2 . gelu(W1 . A + b1) + b2) with the 4C-wide hidden
// activation kept on chip (wgmma + TMA, sm_90a).  Reference op: timm ConvNeXtBlock.mlp (Linear C->4C, GELU, Linear 4C->C)
// * gamma + shortcut (timm 0.6.7, un-vendored), called from models/GDRN_double_mask.py:102 through the backbone.
//
// One persistent CTA per SM, 384 threads: warp 0 lane 0 is the TMA producer, warps 4..11 are two consumer warpgroups
// (rows [0, 64) and [64, 128) of a 128-row tile).  Per tile the A rows stay resident in shared memory and the 512 hidden
// columns are processed in eight chunks of 64:
//   fc1   h[64 x 64] = A . W1[chunk]^T                      (wgmma, registers)
//         + b1, GELU, bf16 -> the warpgroup's rows of the H tile in shared memory, written directly in the
//         128B-swizzled K-major operand layout the TMA would produce
//   fc2   o[64 x 128] += H . W2[:, chunk]^T                  (wgmma, H tile as the A operand, accumulator in registers)
// and after the last chunk every thread adds gamma * (o + b2) to its x elements.  Weight chunks {W1 rows, W2 columns}
// stream through a ring of stages; the weights (256 KB, 512 KB split) stay in L2 across tiles.
// X3 (split-bf16 parity mode): A [M, 2C], W1 [4C, 2C], W2 [C, 8C] hold [hi | lo] halves; every contraction is the three
// products lo.hi + hi.lo + hi.hi of one k-chunk (the order of the X3 GEMM kernel), GELU is the exact erf form and the
// hidden activation is stored as its hi / lo bf16 pair -- the same arithmetic as the two-GEMM path.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "gemm_tc.h"
#include "gemm_epilogue.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BLOCK_K = 64;                       // 64 bf16 = 128 B = one swizzle row
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int MF_C = 128;
constexpr int MF_HC = 64;                         // hidden columns per chunk
constexpr int MF_CHUNKS = 4 * MF_C / MF_HC;       // 8
constexpr int MF_KC1 = MF_C / BLOCK_K;            // k-chunks of fc1 (2)
constexpr int MF_W1_TILE = MF_HC * BLOCK_K * 2;   // 64 rows x 64 k: 8 KB
constexpr int MF_W2_TILE = MF_C * BLOCK_K * 2;    // 128 rows x 64 k: 16 KB

struct MlpPlan {
  CUtensorMap tmap_a;    // A  [M, S*C]   bf16, box {64, 128}
  CUtensorMap tmap_w1;   // W1 [4C, S*C]  bf16, box {64, 64}
  CUtensorMap tmap_w2;   // W2 [C, S*4C]  bf16, box {64, 128}
  const float* b1;       // [4C]
  const float* b2;       // [C]
  const float* gamma;    // [C]
  float* x;              // [M, C] fp32, updated in place
  int m_tiles;
};

template <bool X3>
struct MfCfg {
  static constexpr int S = X3 ? 2 : 1;
  static constexpr int A_BYTES = S * MF_KC1 * A_STAGE_BYTES;            // 32 / 64 KB
  static constexpr int H_BYTES = S * A_STAGE_BYTES;                     // 128 rows x 64 hidden columns: 16 / 32 KB
  static constexpr int STAGE_BYTES = S * (MF_KC1 * MF_W1_TILE + MF_W2_TILE);
  static constexpr int RING = (227 * 1024 - 1024 - 256 - A_BYTES - H_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = RING > 6 ? 6 : RING;
  static constexpr int SMEM_BYTES = A_BYTES + H_BYTES + STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(STAGES >= 2, "fused MLP: shared-memory ring needs two stages");
};

// byte offset of bf16 element (r, c) in a 128B-swizzled K-major tile of 64-column rows (the TMA SWIZZLE_128B layout)
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((c >> 3) ^ (r & 7)) & 7) << 4) + (c & 7) * 2);
}

template <bool X3>
__global__ void __launch_bounds__(NUM_THREADS, 1) mlp_fused_kernel(const __grid_constant__ MlpPlan fp) {
  using C = MfCfg<X3>;
  const uint32_t smem_base = (ptx::smem_u32(gemm_smem) + 1023u) & ~1023u;
  uint8_t* smem_gen = gemm_smem + (smem_base - ptx::smem_u32(gemm_smem));
  const uint32_t a_base = smem_base;                       // [h][kc] tiles of 128 rows x 64 k
  const uint32_t h_base = a_base + C::A_BYTES;             // [h] tiles of 128 rows x 64 hidden columns
  const uint32_t ring_base = h_base + C::H_BYTES;          // stage: [h][kc] W1 tiles, then [h] W2 tiles
  const uint32_t bar_base = ring_base + C::STAGES * C::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
  const uint32_t a_full = bar_base + 8u * (2 * C::STAGES);
  const uint32_t a_empty = a_full + 8u;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  ptx::griddep_launch();
  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&fp.tmap_a);
    ptx::prefetch_tmap(&fp.tmap_w1);
    ptx::prefetch_tmap(&fp.tmap_w2);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);   // one arrive per consumer warpgroup
    }
    ptx::mbar_init(a_full, 1);
    ptx::mbar_init(a_empty, 2);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::griddep_wait();

  if (warp == 0 && lane == 0) {
    // ================= TMA producer =================
    int stage = 0;
    uint32_t phase = 0, aphase = 0;
    for (int tile = blockIdx.x; tile < fp.m_tiles; tile += gridDim.x) {
      ptx::mbar_wait_nocall(a_empty, aphase ^ 1);
      ptx::mbar_arrive_expect_tx(a_full, C::A_BYTES);
      for (int h = 0; h < C::S; ++h)
        for (int kc = 0; kc < MF_KC1; ++kc)
          ptx::tma_load_2d(a_base + (h * MF_KC1 + kc) * A_STAGE_BYTES, &fp.tmap_a, a_full, h * MF_C + kc * BLOCK_K,
                           tile * BLOCK_M);
      aphase ^= 1;
      for (int j = 0; j < MF_CHUNKS; ++j) {
        ptx::mbar_wait_nocall(empty_bar(stage), phase ^ 1);
        const uint32_t sw = ring_base + stage * C::STAGE_BYTES;
        ptx::mbar_arrive_expect_tx(full_bar(stage), C::STAGE_BYTES);
        for (int h = 0; h < C::S; ++h) {
          for (int kc = 0; kc < MF_KC1; ++kc)
            ptx::tma_load_2d(sw + (h * MF_KC1 + kc) * MF_W1_TILE, &fp.tmap_w1, full_bar(stage), h * MF_C + kc * BLOCK_K,
                             j * MF_HC);
          ptx::tma_load_2d(sw + C::S * MF_KC1 * MF_W1_TILE + h * MF_W2_TILE, &fp.tmap_w2, full_bar(stage),
                           h * 4 * MF_C + j * MF_HC, 0);
        }
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ================= consumers =================
    const int ew = warp - 4;
    const int wg = ew >> 2;              // rows [64 wg, 64 wg + 64) of the tile
    const int wl = ew & 3;
    const int bar_id = 2 + wg;           // named barrier of this warpgroup (128 threads)
    const bool leader = (wl == 0 && lane == 0);
    int stage = 0;
    uint32_t phase = 0, aphase = 0;
    for (int tile = blockIdx.x; tile < fp.m_tiles; tile += gridDim.x) {
      ptx::mbar_wait_nocall(a_full, aphase);
      aphase ^= 1;
      float o[MF_C / 2];
#pragma unroll
      for (int i = 0; i < MF_C / 2; ++i) o[i] = 0.f;
      for (int j = 0; j < MF_CHUNKS; ++j) {
        ptx::mbar_wait_nocall(full_bar(stage), phase);
        const uint32_t sw = ring_base + stage * C::STAGE_BYTES;
        // ---- fc1: h = A . W1[chunk]^T (X3: lo.hi + hi.lo + hi.hi per k-chunk) ----
        float hacc[MF_HC / 2];
#pragma unroll
        for (int i = 0; i < MF_HC / 2; ++i) hacc[i] = 0.f;
        ptx::wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < MF_KC1; ++kc) {
#pragma unroll
          for (int q = 0; q < (X3 ? 3 : 1); ++q) {
            const int ah = (X3 && q == 0) ? 1 : 0, bh = (X3 && q == 1) ? 1 : 0;
            const uint64_t ad = ptx::make_sw128_kmajor_desc(a_base + (ah * MF_KC1 + kc) * A_STAGE_BYTES + wg * (A_STAGE_BYTES / 2));
            const uint64_t bd = ptx::make_sw128_kmajor_desc(sw + (bh * MF_KC1 + kc) * MF_W1_TILE);
#pragma unroll
            for (int kk = 0; kk < BLOCK_K / MMA_K; ++kk)
              ptx::Wgmma<MF_HC>::mma(hacc, ad + 2u * kk, bd + 2u * kk, (kc | q | kk) != 0 ? 1u : 0u);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if (j == MF_CHUNKS - 1 && leader) ptx::mbar_arrive(a_empty);   // A of this tile is no longer read
        // ---- + b1, GELU, bf16 (hi / lo) -> this warpgroup's rows of the H tile ----
        ptx::named_bar_sync(bar_id, 128);    // the previous chunk's fc2 of the whole warpgroup has retired
        {
          const int r0 = wg * 64 + wl * 16 + (lane >> 2);
          uint8_t* hgen = smem_gen + (h_base - smem_base);
#pragma unroll
          for (int t = 0; t < MF_HC / 8; ++t) {
            const int c = t * 8 + (lane & 3) * 2;
            const float2 b = __ldg(reinterpret_cast<const float2*>(fp.b1 + j * MF_HC + c));
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int r = r0 + 8 * half;
              const float v0 = hacc[4 * t + 2 * half], v1 = hacc[4 * t + 2 * half + 1];
              if constexpr (X3) {
                f32x2_t v2 = gelu_erf2(f2_add(f2_pack(v0, v1), f2_pack(b.x, b.y)));
                const float2 f = f2_unpack(v2);
                const uint32_t hb = pack_bf16(f.x, f.y);
                const float2 d = f2_unpack(f2_sub(v2, f2_pack(__uint_as_float(hb << 16), __uint_as_float(hb & 0xffff0000u))));
                *reinterpret_cast<uint32_t*>(hgen + sw128_off(r, c)) = hb;
                *reinterpret_cast<uint32_t*>(hgen + A_STAGE_BYTES + sw128_off(r, c)) = pack_bf16(d.x, d.y);
              } else {
                *reinterpret_cast<uint32_t*>(hgen + sw128_off(r, c)) = gelu_pack2_f16(v0 + b.x, v1 + b.y);
              }
            }
          }
        }
        ptx::fence_proxy_async();            // generic-proxy stores -> visible to wgmma (async proxy)
        ptx::named_bar_sync(bar_id, 128);
        // ---- fc2: o += H . W2[:, chunk]^T (X3: lo.hi + hi.lo + hi.hi) ----
        ptx::wgmma_fence();
#pragma unroll
        for (int q = 0; q < (X3 ? 3 : 1); ++q) {
          const int ah = (X3 && q == 0) ? 1 : 0, bh = (X3 && q == 1) ? 1 : 0;
          const uint64_t ad = ptx::make_sw128_kmajor_desc(h_base + ah * A_STAGE_BYTES + wg * (A_STAGE_BYTES / 2));
          const uint64_t bd = ptx::make_sw128_kmajor_desc(sw + C::S * MF_KC1 * MF_W1_TILE + bh * MF_W2_TILE);
#pragma unroll
          for (int kk = 0; kk < BLOCK_K / MMA_K; ++kk)
            ptx::Wgmma<MF_C>::mma(o, ad + 2u * kk, bd + 2u * kk, (j | q | kk) != 0 ? 1u : 0u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        if (leader) ptx::mbar_arrive(empty_bar(stage));
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      // ---- x += gamma * (o + b2): the same rounding as the residual GEMM's L2 reduce-add ----
      const long long r0 = (long long)tile * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2);
#pragma unroll
      for (int t = 0; t < MF_C / 8; ++t) {
        const int c = t * 8 + (lane & 3) * 2;
        const float2 b = __ldg(reinterpret_cast<const float2*>(fp.b2 + c));
        const float2 g = __ldg(reinterpret_cast<const float2*>(fp.gamma + c));
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          float2* xp = reinterpret_cast<float2*>(fp.x + (r0 + 8 * half) * MF_C + c);
          float2 xv = *xp;
          xv.x = __fadd_rn(xv.x, __fmul_rn(g.x, __fadd_rn(o[4 * t + 2 * half], b.x)));
          xv.y = __fadd_rn(xv.y, __fmul_rn(g.y, __fadd_rn(o[4 * t + 2 * half + 1], b.y)));
          *xp = xv;
        }
      }
    }
  }
}

template <bool X3>
int mlp_launch(const void* A, const void* W1, const float* b1, const void* W2, const float* b2, const float* gamma,
               float* x, long long M, cudaStream_t stream) {
  using C = MfCfg<X3>;
  MlpPlan fp;
  memset(&fp, 0, sizeof(fp));
  const uint64_t S = C::S;
  {
    const uint64_t dims[2] = {S * MF_C, (uint64_t)M}, str[1] = {S * MF_C * 2};
    const uint32_t box[2] = {64, 128};
    int rc = make_tmap_bf16(&fp.tmap_a, A, 2, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  {
    const uint64_t dims[2] = {S * MF_C, 4 * MF_C}, str[1] = {S * MF_C * 2};
    const uint32_t box[2] = {64, 64};
    int rc = make_tmap_bf16(&fp.tmap_w1, W1, 2, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  {
    const uint64_t dims[2] = {S * 4 * MF_C, MF_C}, str[1] = {S * 4 * MF_C * 2};
    const uint32_t box[2] = {64, 128};
    int rc = make_tmap_bf16(&fp.tmap_w2, W2, 2, dims, str, box);
    if (rc != GDRN_OK) return rc;
  }
  fp.b1 = b1; fp.b2 = b2; fp.gamma = gamma; fp.x = x;
  fp.m_tiles = (int)(M / BLOCK_M);
  auto kfn = mlp_fused_kernel<X3>;
  GDRN_OPT_IN_SMEM(kfn, C::SMEM_BYTES);
  const int grid = fp.m_tiles < gdrn_num_sms() ? fp.m_tiles : gdrn_num_sms();
  GDRN_CHECK_CUDA(gdrn_launch_dep(kfn, dim3(grid), dim3(NUM_THREADS), C::SMEM_BYTES, stream, fp));
  gdrn_count_launch(1);
  gdrn_record_gemm_kernel(X3 ? GEMM_KERNEL_ID_MLP_FUSED_X3 : GEMM_KERNEL_ID_MLP_FUSED);
  return GDRN_OK;
}

}  // namespace

int mlp_fused_supported(int C, long long M) { return C == MF_C && M % BLOCK_M == 0 && M >= BLOCK_M; }
int mlp_fused_x3_supported(int C, long long M) { return mlp_fused_supported(C, M); }

int mlp_fused_launch(const void* A, const void* W1, const float* b1, const void* W2, const float* b2, const float* gamma,
                     float* x, long long M, int C, cudaStream_t stream) {
  GDRN_REQUIRE(mlp_fused_supported(C, M), "mlp_fused: needs C == 128 and M a positive multiple of 128");
  return mlp_launch<false>(A, W1, b1, W2, b2, gamma, x, M, stream);
}

int mlp_fused_x3_launch(const void* A, const void* W1, const float* b1, const void* W2, const float* b2, const float* gamma,
                        float* x, long long M, int C, cudaStream_t stream) {
  GDRN_REQUIRE(mlp_fused_x3_supported(C, M), "mlp_fused_x3: needs C == 128 and M a positive multiple of 128");
  return mlp_launch<true>(A, W1, b1, W2, b2, gamma, x, M, stream);
}
