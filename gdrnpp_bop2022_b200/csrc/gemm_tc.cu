// wgmma + TMA implicit-GEMM kernel for the GDRNPP dense path (sm_90a).
//
// One persistent CTA per SM, warp-specialised:
//   warp 0 lane 0   : TMA producer  (A pixel boxes + W tiles -> swizzled smem ring)
//   warps 4..11     : two consumer warpgroups.  Warpgroup g issues wgmma m64 x BLOCK_N x 16 (bf16 -> fp32 registers)
//                     for rows [64g, 64g + 64) of the 128-row tile, releases each ring stage as soon as the MMAs that
//                     read it retire, then writes its accumulators into the shared-memory accumulator tile; the same
//                     8 warps then run the fused epilogue from there (gemm_epilogue.cuh) while the producer already
//                     fills the ring for the next tile.  Split-bf16 plain-row GELU / RESID / fp32 STORE GEMMs (REG) skip
//                     the tile: every warp runs the epilogue on its own fragments, and the ring takes the tile's bytes.
// X3 (split-bf16, 64- / 128-wide tiles): a stage holds {A hi, A lo, W hi, W lo} of one k-chunk (32 wide for convolutions,
// 64 for plain rows) and feeds all three products.
// The kernel makes no function call: any call makes ptxas serialize the wgmma pipeline (C7510).
//
// It replaces, for the reference forward (core/gdrn_modeling/models/GDRN_double_mask.py:102-160), every
// cuDNN/cuBLAS call made by timm ConvNeXt (Linear fc1/fc2, stem 4x4s4, 2x2s2 downsample), by the geometry
// head (heads/top_down_doublemask_xyz_region_head.py:177-211: ConvTranspose2d, six 3x3 convs, 1x1 out
// conv) and by ConvPnPNet (heads/conv_pnp_net.py:120-183: three 3x3 s2 convs and four Linear layers).
#include <stdio.h>
#include "gemm_tc.h"
#include "gemm_epilogue.cuh"
#include "wgmma.cuh"

namespace {

// X3: split-bf16 operands with the shared four-tile stage {A hi, A lo, W hi, W lo} of one (tap, k-chunk) feeding the three
// products A_lo*W_hi + A_hi*W_lo + A_hi*W_hi (4 operand tiles per 3 MMA groups instead of 6 with an expanded tap list).
// BK: k-chunk width (bf16 elements) of one ring stage.  64 = 128-byte rows (SWIZZLE_128B); 32 = 64-byte rows
// (SWIZZLE_64B), X3 only: half the bytes per stage, twice the ring depth (gemm_tc_launch picks it, see there).
// REG: the epilogue runs straight from the wgmma registers (epilogue_regs), so there is no shared-memory accumulator tile
// and its bytes go to the ring (split-bf16 plain rows with 64-wide chunks only).
template <int BLOCK_N, bool X3, int BK = 64, bool REG = false>
struct Cfg {
  static_assert(BK == 64 || (X3 && BK == 32), "gemm: 32-wide k-chunks exist for the split-bf16 kernel only");
  static_assert(!REG || (X3 && BK == 64), "gemm: the register epilogue exists for the 64-wide split-bf16 kernel only");
  static constexpr int BLOCK_K = BK;
  static constexpr int NOPS = X3 ? 2 : 1;  // hi (and lo) copies of each operand per stage
  static constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_TILE_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int B_STAGE_BYTES = NOPS * B_TILE_BYTES;
  static constexpr int A_BYTES = NOPS * A_TILE_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_STAGE_BYTES;
  static constexpr int ACC_BYTES = REG ? 0 : acc_bytes<BLOCK_N>();
  static constexpr int RING = (SMEM_BUDGET - ACC_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = RING > 8 ? 8 : RING;
  static constexpr int SMEM_BYTES = ACC_BYTES + STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + NUM_EPI_WARPS * EPI_STAGE_BYTES;
  // L2 prefetch distance of A: 384 k-elements ahead of the ring, whatever the chunk width
  static constexpr int PREFETCH_AHEAD = 384 / BLOCK_K;
  static_assert(STAGES >= 2, "gemm: shared-memory ring needs two stages");
  // every tile start (stage, hi / lo half, warpgroup half of A) stays on a swizzle atom (1024 B / 512 B)
  static_assert(ACC_BYTES % 1024 == 0 && STAGE_BYTES % 1024 == 0 && A_TILE_BYTES % 1024 == 0 && B_TILE_BYTES % 1024 == 0,
                "gemm: operand tiles must keep the swizzle-atom alignment");
};
// the 32-wide X3 kernel consumes its stages in pairs (one 64-wide k-step): at BLOCK_N = 128 two more stages load meanwhile
static_assert(Cfg<128, true, 32>::STAGES >= 4, "gemm: the 32-wide split-bf16 128-wide kernel needs a four-deep operand ring");
static_assert(Cfg<64, true, 32>::STAGES >= 6, "gemm: the 32-wide split-bf16 64-wide kernel needs a six-deep operand ring");
// without the accumulator tile the 64-wide split-bf16 ring gains a stage: 3 x 64 KB at BLOCK_N = 128, 4 x 48 KB at 64
static_assert(Cfg<128, true, 64, true>::STAGES >= 3, "gemm: the register-epilogue split-bf16 128-wide kernel needs a three-deep operand ring");
static_assert(Cfg<64, true, 64, true>::STAGES >= 4, "gemm: the register-epilogue split-bf16 64-wide kernel needs a four-deep operand ring");

constexpr int CONSUMER_THREADS = 256;
constexpr int BAR_ACC = 1;         // named barrier of the two consumer warpgroups (accumulator tile hand-over)

template <int BLOCK_N, int EPI, bool X3, int BK, bool REG>
__global__ void __launch_bounds__(NUM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ GemmPlan p) {
  using C = Cfg<BLOCK_N, X3, BK, REG>;
  // 1024-byte alignment required by SWIZZLE_128B: [accumulator tile | ring | epilogue staging | barriers]
  const uint32_t smem_base = (ptx::smem_u32(gemm_smem) + 1023u) & ~1023u;
  const uint32_t ring_base = smem_base + C::ACC_BYTES;
  const uint32_t bar_base = ring_base + C::STAGES * C::STAGE_BYTES + NUM_EPI_WARPS * EPI_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
  uint8_t* smem_gen = gemm_smem + (smem_base - ptx::smem_u32(gemm_smem));
  float* acc_smem = reinterpret_cast<float*>(smem_gen);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // epilogues that need the whole row in one thread (LayerNorm, out-conv) or tiny N keep 4 warps + direct stores
  constexpr bool kStaged = (BLOCK_N >= 64) && (EPI == EPI_STORE || EPI == EPI_GELU || EPI == EPI_RESID || EPI == EPI_GNSTATS);
  uint8_t* stage_base = smem_gen + C::ACC_BYTES + C::STAGES * C::STAGE_BYTES;  // 1024-aligned (TMA-store tiles are 128B-swizzled)

  ptx::griddep_launch();
  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&p.tmap_a);
    ptx::prefetch_tmap(&p.tmap_b);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::griddep_wait();

  const int total_tiles = p.m_tiles * p.n_tiles;
  const int k_iters = p.num_taps * p.k_chunks;

  // REG: the consumers keep their accumulators live through the epilogue, so they take the registers the producer
  // warpgroup does not use (setmaxnreg is per warpgroup: warps 1..3 and lanes 1..31 of warp 0 lower theirs too)
  if (warp < 4) {
    if constexpr (REG) ptx::setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ================= TMA producer =================
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_tile = tile % p.n_tiles;
        const int m_tile = tile / p.n_tiles;
        int x0 = 0, y0 = 0, b0 = 0;
        if (p.a_rank != 2) {
          int tx = m_tile % p.tiles_x;
          int t2 = m_tile / p.tiles_x;
          x0 = tx << p.lg_bw;
          y0 = (t2 % p.tiles_y) << p.lg_bh;
          b0 = (t2 / p.tiles_y) << p.lg_bb;
        }
        int brow = n_tile * BLOCK_N;
        if (EPI == EPI_OUTCONV) {
          long long grow = (long long)m_tile * BLOCK_M;
          int b = (int)(grow / p.rows_per_roi);
          int cls = p.roi_classes ? (int)p.roi_classes[b] : 0;   // NULL: class-agnostic head (one slab)
          cls = cls < 0 ? 0 : (cls >= p.num_classes ? p.num_classes - 1 : cls);  // never index outside the weights
          brow += cls * p.b_rows_per_class;
        }
        for (int tap = 0; tap < p.num_taps; ++tap) {
          const GemmTap tp = p.taps[tap];
          for (int kc = 0; kc < p.k_chunks; ++kc) {
            ptx::mbar_wait_nocall(empty_bar(stage), phase ^ 1);
            const uint32_t sa = ring_base + stage * C::STAGE_BYTES;
            const uint32_t sb = sa + C::A_BYTES;
            ptx::mbar_arrive_expect_tx(full_bar(stage), C::STAGE_BYTES);
            const int k0 = kc * C::BLOCK_K;
#pragma unroll
            for (int h = 0; h < C::NOPS; ++h) {   // h = 1: the lo halves, behind the hi tiles of the stage
              const uint32_t da = sa + h * C::A_TILE_BYTES;
              const int ca = k0 + tp.c0 + h * p.x3_a_lo;
              if (p.a_rank == 2) {
                ptx::tma_load_2d(da, &p.tmap_a, full_bar(stage), ca, m_tile * BLOCK_M + tp.d1);
              } else if (p.a_rank == 4) {
                ptx::tma_load_4d(da, &p.tmap_a, full_bar(stage), ca, x0 + tp.d1, y0 + tp.d2, b0);
              } else {
                ptx::tma_load_5d(da, &p.tmap_a, full_bar(stage), ca, x0 + tp.d1, tp.d2, y0 + tp.d3, b0);
              }
              ptx::tma_load_2d(sb + h * C::B_TILE_BYTES, &p.tmap_b, full_bar(stage), tp.b_off + k0 + h * p.x3_b_lo, brow);
            }
            if (p.a_rank == 2) {
              // A is streamed from HBM (it was written by the previous kernel): request it into L2 several
              // k-iterations ahead so the shared-memory ring only has to cover L2 latency, not DRAM latency.
              int pk = kc + C::PREFETCH_AHEAD, pm = m_tile;
              if (pk >= p.k_chunks) {
                pk -= p.k_chunks;
                const int nt = tile + gridDim.x;
                const int nm = nt / p.n_tiles;
                pm = (nt < total_tiles && nm != m_tile) ? nm : -1;
              }
              if (pm >= 0 && pk < p.k_chunks && p.num_taps == 1) ptx::tma_prefetch_2d(&p.tmap_a, pk * C::BLOCK_K, pm * BLOCK_M);
            }
            if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    if constexpr (REG) ptx::setmaxnreg_inc<232>();
    // ================= consumers: wgmma mainloop, accumulator hand-over, epilogue =================
    const int ew = warp - 4;
    const int wg = ew >> 2;             // rows [64 wg, 64 wg + 64) of the tile
    const int wl = ew & 3;              // warp inside the warpgroup
    int stage = 0;
    uint32_t phase = 0;
    uint32_t sbuf = 0;  // REG, EPI_GELU: chunks this warp has TMA-stored (picks the half of its staging slot)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_tile = tile % p.n_tiles;
      const int m_tile = tile / p.n_tiles;
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      if constexpr (X3 && BK == 32) {
        // Two 32-wide stages make one 64-wide k-step, issued as A_lo*W_hi, A_hi*W_lo, A_hi*W_hi over all 64 k -- small
        // terms first, and the fp32 summation order of a 64-wide stage -- in four commit groups, so that the first stage
        // is released as soon as its last product (hi*hi) retires, while the second one's hi*hi still runs.
        for (int k = 0; k < k_iters; k += 2) {
          const int s0 = stage;
          const uint32_t ph0 = phase;
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
          const int s1 = stage;
          const uint32_t ph1 = phase;
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
          const uint32_t a0 = ring_base + s0 * C::STAGE_BYTES + wg * (C::A_TILE_BYTES / 2);
          const uint32_t b0 = ring_base + s0 * C::STAGE_BYTES + C::A_BYTES;
          const uint32_t a1 = ring_base + s1 * C::STAGE_BYTES + wg * (C::A_TILE_BYTES / 2);
          const uint32_t b1 = ring_base + s1 * C::STAGE_BYTES + C::A_BYTES;
          // one product over a 32-wide stage: two k16 steps, +32 B (+2 in the (addr >> 4) field) inside the swizzle row
          auto mma32 = [&](uint32_t a, uint32_t b, uint32_t accumulate) {
            const uint64_t ad = ptx::make_sw64_kmajor_desc(a), bd = ptx::make_sw64_kmajor_desc(b);
            ptx::Wgmma<BLOCK_N>::mma(acc, ad, bd, accumulate);
            ptx::Wgmma<BLOCK_N>::mma(acc, ad + 2u, bd + 2u, 1u);
          };
          ptx::mbar_wait_nocall(full_bar(s0), ph0);
          ptx::wgmma_fence();
          mma32(a0 + C::A_TILE_BYTES, b0, k != 0 ? 1u : 0u);                  // lo*hi, k [0, 32)
          ptx::wgmma_commit();
          // the previous k-step's last group has retired: release its second stage
          ptx::wgmma_wait<1>();
          if (prev_stage >= 0 && wl == 0 && lane == 0) ptx::mbar_arrive(empty_bar(prev_stage));
          ptx::mbar_wait_nocall(full_bar(s1), ph1);
          ptx::wgmma_fence();
          mma32(a1 + C::A_TILE_BYTES, b1, 1u);                                // lo*hi, k [32, 64)
          mma32(a0, b0 + C::B_TILE_BYTES, 1u);                                // hi*lo, k [0, 32)
          ptx::wgmma_commit();
          mma32(a1, b1 + C::B_TILE_BYTES, 1u);                                // hi*lo, k [32, 64)
          mma32(a0, b0, 1u);                                                  // hi*hi, k [0, 32): last read of s0
          ptx::wgmma_commit();
          mma32(a1, b1, 1u);                                                  // hi*hi, k [32, 64)
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();
          if (wl == 0 && lane == 0) ptx::mbar_arrive(empty_bar(s0));
          prev_stage = s1;
        }
      } else {
        for (int k = 0; k < k_iters; ++k) {
          ptx::mbar_wait_nocall(full_bar(stage), phase);
          const uint32_t sa = ring_base + stage * C::STAGE_BYTES + wg * (C::A_TILE_BYTES / 2);
          const uint32_t sb = ring_base + stage * C::STAGE_BYTES + C::A_BYTES;
          ptx::wgmma_fence();
          // X3: (A lo, W hi), (A hi, W lo), (A hi, W hi) -- small terms first; otherwise the single (A, W) product
#pragma unroll
          for (int q = 0; q < (X3 ? 3 : 1); ++q) {
            const uint32_t a_off = (X3 && q == 0) ? C::A_TILE_BYTES : 0u;
            const uint32_t b_off = (X3 && q == 1) ? C::B_TILE_BYTES : 0u;
            const uint64_t adesc = ptx::make_sw128_kmajor_desc(sa + a_off);
            const uint64_t bdesc = ptx::make_sw128_kmajor_desc(sb + b_off);
#pragma unroll
            for (int kk = 0; kk < C::BLOCK_K / MMA_K; ++kk) {
              // advance 16 bf16 = 32 B inside the 128B swizzle row: +2 in the (addr >> 4) field
              ptx::Wgmma<BLOCK_N>::mma(acc, adesc + 2u * kk, bdesc + 2u * kk, (k | q | kk) != 0 ? 1u : 0u);
            }
          }
          ptx::wgmma_commit();
          // the previous stage's MMAs have retired once at most this stage's group is in flight: release that slot
          ptx::wgmma_wait<1>();
          if (prev_stage >= 0 && wl == 0 && lane == 0) ptx::mbar_arrive(empty_bar(prev_stage));
          prev_stage = stage;
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
      float2 xres[REG && EPI == EPI_RESID ? BLOCK_N / 4 : 1];
      if constexpr (REG && EPI == EPI_RESID) frag_resid_load<BLOCK_N>(p, m_tile, n_tile, wg * 64 + wl * 16, lane, xres);
      ptx::wgmma_wait<0>();
      if (prev_stage >= 0 && wl == 0 && lane == 0) ptx::mbar_arrive(empty_bar(prev_stage));
      if constexpr (REG) {
        epilogue_regs<BLOCK_N, EPI>(p, m_tile, n_tile, wg * 64 + wl * 16, lane, acc, xres, stage_base + ew * EPI_STAGE_BYTES,
                                    sbuf);
        continue;
      }

      if (kStaged && EPI != EPI_GNSTATS && !p.use_tma_store) {
        // this warp's bias (and layer-scale gamma) segment -> its shared-memory slot
        float* sbw = reinterpret_cast<float*>(stage_base + ew * EPI_STAGE_BYTES + 32 * EPI_STAGE_PITCH + 256);
        const int cb = n_tile * BLOCK_N + (ew >> 2) * (BLOCK_N / 2) + lane * 4;
        if (lane * 4 < BLOCK_N / 2) {
          float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f), g4 = b4;
          if (cb + 3 < p.N) {
            if (p.bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + cb));
            if (EPI == EPI_RESID) g4 = __ldg(reinterpret_cast<const float4*>(p.gamma + cb));
          }
          *reinterpret_cast<float4*>(sbw + lane * 4) = b4;
          if (EPI == EPI_RESID) *reinterpret_cast<float4*>(sbw + 128 + lane * 4) = g4;
        }
        __syncwarp();
      }
      // the previous tile's epilogue has finished reading the accumulator tile
      ptx::named_bar_sync(BAR_ACC, CONSUMER_THREADS);
      {
        const int r0 = wg * 64 + wl * 16 + (lane >> 2);
        const int c0 = (lane & 3) * 2;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          *reinterpret_cast<float2*>(acc_smem + acc_index<BLOCK_N>(r0, j * 8 + c0)) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(acc_smem + acc_index<BLOCK_N>(r0 + 8, j * 8 + c0)) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      ptx::named_bar_sync(BAR_ACC, CONSUMER_THREADS);
      if constexpr (kStaged) {
        epilogue_tile_staged<BLOCK_N, EPI>(p, m_tile, n_tile, 0u, ew, lane, stage_base + ew * EPI_STAGE_BYTES);
      } else if (ew < 4) {
        const uint32_t acc_row = (uint32_t)(ew * 32) << 16;
        epilogue_tile<BLOCK_N, EPI>(p, m_tile, n_tile, acc_row, lane, stage_base + ew * EPI_STAGE_BYTES);
      }
    }
    if (lane == 0) ptx::bulk_wait0();  // outstanding TMA stores (no-op when none were issued)
  }
}

// Every kernel gemm_tc_launch can launch, numbered for the launch record (gdrn_gemm_kernels_launched).  The order is the
// ABI of that record: append, never reorder (the Python side names the bits from the same list, _lib.GEMM_KERNELS).
struct GemmKernelKey {
  int block_n, epi;
  bool x3;
  int bk;
  bool reg;
};
constexpr GemmKernelKey kGemmKernels[] = {
    // bf16
    {128, EPI_GELU, false, 64, false},
    {128, EPI_RESID, false, 64, false},
    {128, EPI_STORE, false, 64, false},
    {128, EPI_GNSTATS, false, 64, false},
    {128, EPI_BIAS_LN, false, 64, false},
    {64, EPI_GELU, false, 64, false},
    {64, EPI_RESID, false, 64, false},
    {64, EPI_STORE, false, 64, false},
    {64, EPI_GNSTATS, false, 64, false},
    {16, EPI_STORE, false, 64, false},
    {80, EPI_OUTCONV, false, 64, false},
    // split-bf16, register epilogue
    {128, EPI_GELU, true, 64, true},
    {128, EPI_RESID, true, 64, true},
    {128, EPI_STORE, true, 64, true},
    {64, EPI_GELU, true, 64, true},
    {64, EPI_RESID, true, 64, true},
    {64, EPI_STORE, true, 64, true},
    // split-bf16 stem and convolutions
    {128, EPI_BIAS_LN, true, 64, false},
    {128, EPI_GNSTATS, true, 32, false},
    {64, EPI_GNSTATS, true, 32, false},
};
static_assert(sizeof(kGemmKernels) / sizeof(kGemmKernels[0]) == GEMM_NUM_TC_KERNELS, "gemm: kGemmKernels size");

constexpr bool same_kernel(const GemmKernelKey& a, const GemmKernelKey& b) {
  return a.block_n == b.block_n && a.epi == b.epi && a.x3 == b.x3 && a.bk == b.bk && a.reg == b.reg;
}
constexpr bool gemm_kernels_unique() {
  for (int i = 0; i < GEMM_NUM_TC_KERNELS; ++i)
    for (int j = i + 1; j < GEMM_NUM_TC_KERNELS; ++j)
      if (same_kernel(kGemmKernels[i], kGemmKernels[j])) return false;
  return true;
}
static_assert(gemm_kernels_unique(), "gemm: an instantiation is listed twice in kGemmKernels");

template <int BLOCK_N, int EPI, bool X3, int BK, bool REG>
constexpr int gemm_kernel_id() {
  for (int i = 0; i < GEMM_NUM_TC_KERNELS; ++i)
    if (same_kernel(kGemmKernels[i], GemmKernelKey{BLOCK_N, EPI, X3, BK, REG})) return i;
  return -1;
}

template <int BLOCK_N, int EPI, bool X3 = false, int BK = 64, bool REG = false>
int launch_inst(const GemmPlan& plan, cudaStream_t stream) {
  using C = Cfg<BLOCK_N, X3, BK, REG>;
  constexpr int kId = gemm_kernel_id<BLOCK_N, EPI, X3, BK, REG>();
  static_assert(kId >= 0, "gemm: every instantiation needs an entry in kGemmKernels");
  auto kfn = gemm_tc_kernel<BLOCK_N, EPI, X3, BK, REG>;
  GDRN_OPT_IN_SMEM(kfn, C::SMEM_BYTES);
  int total = plan.m_tiles * plan.n_tiles;
  if (total <= 0) return GDRN_OK;
  int grid = total < gdrn_num_sms() ? total : gdrn_num_sms();
  GDRN_CHECK_CUDA(gdrn_launch_dep(kfn, dim3(grid), dim3(NUM_THREADS), C::SMEM_BYTES, stream, plan));
  gdrn_count_launch(1);
  gdrn_record_gemm_kernel(kId);
  return GDRN_OK;
}

}  // namespace

int gemm_tc_launch(const GemmPlan& plan_in, int block_n, cudaStream_t stream) {
  GemmPlan plan = plan_in;
  GDRN_REQUIRE(plan.a_rank == 2 || plan.a_rank == 4 || plan.a_rank == 5, "gemm: bad a_rank");
  GDRN_REQUIRE(plan.a_ptr != nullptr && plan.b_ptr != nullptr && plan.a_k > 0, "gemm: plan without operands");
  plan.use_tma_store = 0;
  plan.resid_reduce = 0;
  if (block_n > 128) {
    // 128 x 256 tiles would need a 128 KB accumulator tile next to the operand ring: run them as two 128-wide tiles
    block_n = 128;
    plan.n_tiles = (plan.N + block_n - 1) / block_n;
  }
  // split-bf16 (x3): taps[] lists the hi operands.  64- / 128-wide tiles run the shared four-tile stage (X3 kernel); the
  // other widths (the 80-wide out-conv) expand every tap to (A lo, W hi) + (A hi, W lo) + (A hi, W hi), small terms first.
  const bool x3_shared = plan.split && (block_n == 64 || block_n == 128) && plan.epi != EPI_OUTCONV;
  if (plan.split && !x3_shared) {
    GDRN_REQUIRE(plan.num_taps >= 1 && 3 * plan.num_taps <= GEMM_MAX_TAPS, "gemm: bad num_taps (split)");
    const int n = plan.num_taps;
    for (int t = n - 1; t >= 0; --t) {
      const GemmTap h = plan.taps[t];
      GemmTap al = h; al.c0 += plan.x3_a_lo;
      GemmTap bl = h; bl.b_off += plan.x3_b_lo;
      plan.taps[t] = al; plan.taps[n + t] = bl; plan.taps[2 * n + t] = h;
    }
    plan.num_taps = 3 * n;
  }
  // k-chunk width.  Split-bf16 convolutions (rank-4/5 pixel boxes, A re-read from L2 by every tap) run 32-wide chunks: the
  // deeper ring covers their L2 round trips.  Plain rank-2 rows keep 64-wide chunks: they stream A from HBM, where 128-byte
  // rows beat 64-byte ones (DESIGN §4.1, §7).
  const int bk = (x3_shared && plan.a_rank != 2) ? 32 : 64;
  {  // operand maps at that width
    GDRN_REQUIRE(!x3_shared || plan.a_k % 64 == 0, "gemm: split-bf16 K per tap must be a multiple of 64");
    plan.a_box[0] = (uint32_t)bk;
    int rc = make_tmap_bf16(&plan.tmap_a, plan.a_ptr, plan.a_rank, plan.a_dims, plan.a_str, plan.a_box);
    if (rc != GDRN_OK) return rc;
    const uint64_t dims[2] = {(uint64_t)plan.b_ktot, (uint64_t)plan.b_rows};
    const uint64_t str[1] = {(uint64_t)plan.b_ktot * 2};
    const uint32_t box[2] = {(uint32_t)bk, (uint32_t)block_n};
    rc = make_tmap_bf16(&plan.tmap_b, plan.b_ptr, 2, dims, str, box);
    if (rc != GDRN_OK) return rc;
    plan.k_chunks = (plan.a_k + bk - 1) / bk;
  }
  {
    // bf16 rank-2 rows in 128-wide tiles leave through TMA stores when the output is aligned for them; an in-place
    // residual becomes an L2 reduce-add (x is never read by the SM), an out-of-place one a read-modify-write
    const bool f32 = plan.epi == EPI_RESID || plan.epi == EPI_BIAS_LN || (plan.epi == EPI_STORE && plan.out_f32);
    if (plan.a_rank == 2 && !plan.split && block_n >= 128 && plan.N % 64 == 0 &&
        (plan.epi == EPI_STORE || plan.epi == EPI_GELU || plan.epi == EPI_RESID || plan.epi == EPI_BIAS_LN) &&
        ((uintptr_t)plan.out % 16 == 0) && ((plan.ldo * (f32 ? 4 : 2)) % 16 == 0) &&
        (plan.epi != EPI_RESID || ((uintptr_t)plan.resid % 16 == 0))) {
      const uint64_t dims[2] = {(uint64_t)plan.ldo, (uint64_t)plan.M};
      const uint64_t str[1] = {(uint64_t)plan.ldo * (f32 ? 4 : 2)};
      const uint32_t box[2] = {f32 ? 32u : 64u, 32u};
      int rc = make_tmap_store(&plan.tmap_out, plan.out, f32 ? 1 : 0, dims, str, box);
      if (rc != GDRN_OK) return rc;
      plan.use_tma_store = 1;
      plan.resid_reduce = (plan.epi == EPI_RESID && plan.resid == plan.out) ? 1 : 0;
    }
  }
  // Split-bf16 plain rows with an element-wise epilogue (the ConvNeXt MLPs and downsamples) run it straight from the wgmma
  // registers: without the accumulator tile the operand ring is one stage deeper (DESIGN §4.1).  The split GELU output
  // [hi N | lo N] leaves through TMA stores of 16-row x 64-byte tiles, which need N % 64 == 0 and 16-byte aligned rows.
  const bool reg_epi = x3_shared && plan.a_rank == 2 &&
                       (plan.epi == EPI_RESID || (plan.epi == EPI_STORE && plan.out_f32) || plan.epi == EPI_GELU);
  if (reg_epi && plan.epi == EPI_GELU) {
    GDRN_REQUIRE(plan.N % 64 == 0 && (uintptr_t)plan.out % 16 == 0 && (plan.ldo * 2) % 16 == 0,
                 "gemm: the split-bf16 GELU output needs N % 64 == 0 and a 16-byte aligned out and row pitch");
    const uint64_t dims[2] = {(uint64_t)plan.ldo, (uint64_t)plan.M};
    const uint64_t str[1] = {(uint64_t)plan.ldo * 2};
    const uint32_t box[2] = {32u, 16u};
    int rc = make_tmap_store_plain(&plan.tmap_out, plan.out, 0, dims, str, box);
    if (rc != GDRN_OK) return rc;
    plan.use_tma_store = 1;
  }
  GDRN_REQUIRE(plan.num_taps >= 1 && plan.num_taps <= GEMM_MAX_TAPS, "gemm: bad num_taps");
  if (x3_shared) {
#define GDRN_GEMM_CASE_REG(BN, E) \
  if (reg_epi && block_n == BN && plan.epi == E) return launch_inst<BN, E, true, 64, true>(plan, stream);
    GDRN_GEMM_CASE_REG(128, EPI_GELU)
    GDRN_GEMM_CASE_REG(128, EPI_RESID)
    GDRN_GEMM_CASE_REG(128, EPI_STORE)
    GDRN_GEMM_CASE_REG(64, EPI_GELU)
    GDRN_GEMM_CASE_REG(64, EPI_RESID)
    GDRN_GEMM_CASE_REG(64, EPI_STORE)
#undef GDRN_GEMM_CASE_REG
    // the stem (rank-2 rows, LayerNorm epilogue) and the convolutions (32-wide chunks, GroupNorm sums)
    if (bk == 64 && block_n == 128 && plan.epi == EPI_BIAS_LN) return launch_inst<128, EPI_BIAS_LN, true, 64>(plan, stream);
    if (bk == 32 && block_n == 128 && plan.epi == EPI_GNSTATS) return launch_inst<128, EPI_GNSTATS, true, 32>(plan, stream);
    if (bk == 32 && block_n == 64 && plan.epi == EPI_GNSTATS) return launch_inst<64, EPI_GNSTATS, true, 32>(plan, stream);
  } else {
#define GDRN_GEMM_CASE(BN, E) \
  if (block_n == BN && plan.epi == E) return launch_inst<BN, E>(plan, stream);
    GDRN_GEMM_CASE(128, EPI_GELU)
    GDRN_GEMM_CASE(128, EPI_RESID)
    GDRN_GEMM_CASE(128, EPI_STORE)
    GDRN_GEMM_CASE(128, EPI_GNSTATS)
    GDRN_GEMM_CASE(128, EPI_BIAS_LN)
    GDRN_GEMM_CASE(64, EPI_GELU)
    GDRN_GEMM_CASE(64, EPI_RESID)
    GDRN_GEMM_CASE(64, EPI_STORE)
    GDRN_GEMM_CASE(64, EPI_GNSTATS)
    GDRN_GEMM_CASE(16, EPI_STORE)
    GDRN_GEMM_CASE(80, EPI_OUTCONV)
#undef GDRN_GEMM_CASE
  }
  gdrn_set_last_error(__FILE__, __LINE__, "gemm: unsupported (block_n, epilogue) combination");
  return GDRN_ERR_INVALID;
}

// ------------------------------------------------------------------------------------------------
// Tensor maps (driver entry point resolved at run time: the library does not link libcuda).
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

int make_tmap_f32_plain(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box) {
  PFN_encodeTiled fn = get_encode_fn();
  GDRN_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[160];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(f32) failed: CUresult %d", (int)r);
    gdrn_set_last_error(__FILE__, __LINE__, msg);
    return GDRN_ERR_CUDA;
  }
  return GDRN_OK;
}

// rank-2 output map for the TMA-store epilogue: 128-byte rows, SWIZZLE_128B
int make_tmap_store(CUtensorMap* out, const void* base, int is_f32, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box) {
  PFN_encodeTiled fn = get_encode_fn();
  GDRN_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  cuuint64_t gdim[2] = {dims[0], dims[1]};
  cuuint64_t gstr[1] = {strides_bytes[0]};
  cuuint32_t bx[2] = {box[0], box[1]};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(out, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[160];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(store) failed: CUresult %d (dims %llu,%llu)", (int)r,
             (unsigned long long)dims[0], (unsigned long long)dims[1]);
    gdrn_set_last_error(__FILE__, __LINE__, msg);
    return GDRN_ERR_CUDA;
  }
  return GDRN_OK;
}

int make_tmap_store_plain(CUtensorMap* out, const void* base, int is_f32, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box) {
  PFN_encodeTiled fn = get_encode_fn();
  GDRN_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  cuuint64_t gdim[2] = {dims[0], dims[1]};
  cuuint64_t gstr[1] = {strides_bytes[0]};
  cuuint32_t bx[2] = {box[0], box[1]};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(out, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  (box[0] * (is_f32 ? 4 : 2) == 64) ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[160];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(store, plain) failed: CUresult %d (dims %llu,%llu)", (int)r,
             (unsigned long long)dims[0], (unsigned long long)dims[1]);
    gdrn_set_last_error(__FILE__, __LINE__, msg);
    return GDRN_ERR_CUDA;
  }
  return GDRN_OK;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
  PFN_encodeTiled fn = get_encode_fn();
  GDRN_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  GDRN_REQUIRE(box[0] == 64 || box[0] == 32, "make_tmap_bf16: k-chunk box must be 64 or 32 elements");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, box[0] == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[160];
    snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r,
             rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    gdrn_set_last_error(__FILE__, __LINE__, msg);
    return GDRN_ERR_CUDA;
  }
  return GDRN_OK;
}
