// Shared device/host helpers for libgdrn_b200.so (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/gdrn_b200.h"

#define GDRN_CHECK_CUDA(expr)                                                                   \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      (void)cudaGetLastError(); /* clear the non-sticky error state */                          \
      gdrn_set_last_error(__FILE__, __LINE__, cudaGetErrorString(_e));                          \
      return GDRN_ERR_CUDA;                                                                     \
    }                                                                                           \
  } while (0)

#define GDRN_REQUIRE(cond, msg)                                                                 \
  do {                                                                                          \
    if (!(cond)) {                                                                              \
      gdrn_set_last_error(__FILE__, __LINE__, msg);                                             \
      return GDRN_ERR_INVALID;                                                                  \
    }                                                                                           \
  } while (0)

void gdrn_set_last_error(const char* file, int line, const char* msg);
void gdrn_count_launch(int n);  // bumps the counter behind gdrn_launch_count()
void gdrn_record_gemm_kernel(int id);  // sets bit id of the record behind gdrn_gemm_kernels_launched()

// The dynamic-shared-memory opt-in and the SM count are PER DEVICE: cache them per device ordinal so that a process
// that drives several GPUs (GdrnPredictor(device="cuda:1"), one engine per device) configures each of them.
constexpr int GDRN_MAX_DEVICES = 64;
static inline int gdrn_cur_device() {
  int d = 0;
  cudaGetDevice(&d);
  return d < 0 ? 0 : (d >= GDRN_MAX_DEVICES ? GDRN_MAX_DEVICES - 1 : d);
}
static inline int gdrn_num_sms() {
  static int n[GDRN_MAX_DEVICES] = {};
  const int dev = gdrn_cur_device();
  if (n[dev] == 0) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}
// once per (kernel instantiation, device): cudaFuncSetAttribute(MaxDynamicSharedMemorySize)
#define GDRN_OPT_IN_SMEM(kfn, bytes)                                                                             \
  do {                                                                                                           \
    static bool gdrn_done_[GDRN_MAX_DEVICES] = {};                                                               \
    const int gdrn_dev_ = gdrn_cur_device();                                                                     \
    if (!gdrn_done_[gdrn_dev_]) {                                                                                \
      GDRN_CHECK_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));     \
      gdrn_done_[gdrn_dev_] = true;                                                                              \
    }                                                                                                            \
  } while (0)


// ---- programmatic dependent launch (PDL) ----
// Every kernel of the per-ROI step is launched with cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's
// CTAs are placed on SMs as the previous kernel's CTAs retire and run their prologue (barrier init,
// tensor-map prefetch, filter-tap loads) under the previous kernel's tail; ptx::griddep_wait() then holds them until the
// previous grid has completed and flushed.  CONTRACT: a kernel launched through gdrn_launch_dep() executes
// ptx::griddep_launch() first and ptx::griddep_wait() in EVERY thread before its first access to global memory that another
// kernel of the stream writes or reads (and before any early return), so that completion stays transitive along the chain.
// Works under stream capture (programmatic graph edges).  GDRN_PDL=0: plain stream-ordered launches.
inline bool gdrn_pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("GDRN_PDL"); v = e ? atoi(e) : 1; }
  return v != 0;
}
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t gdrn_launch_dep(void (*kfn)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int n = 0;
  if (gdrn_pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kfn, static_cast<KArgs>(args)...);
}
#endif

#ifdef __CUDACC__
namespace ptx {

// PDL (see gdrn_launch_dep): let the dependent grid start its prologue / wait for the prerequisite grid's results
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred)::"memory");
  return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded wait: a protocol bug traps (error return to the host) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  int spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins == 64) t0 = clock64();
    if (spins > 64 && (clock64() - t0) > 4000000000LL) {
      printf("gdrn: mbarrier wait timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar,
             parity);
      __trap();
    }
  }
}

// The same bound without the printf, for kernels that issue wgmma: any function call in such a kernel makes ptxas
// serialize the wgmma pipeline (C7510).  A protocol bug still traps.
__device__ __forceinline__ void mbar_wait_nocall(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  int spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins == 64) t0 = clock64();
    if (spins > 64 && (clock64() - t0) > 4000000000LL) asm volatile("trap;");
  }
}

// Bounded cluster-scope acquire wait on a barrier of THIS CTA that peers complete with st.async transaction bytes.
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  int spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins == 64) t0 = clock64();
    if (spins > 64 && (clock64() - t0) > 4000000000LL) {
      printf("gdrn: cluster mbarrier wait timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar,
             parity);
      __trap();
    }
  }
}
// 8-byte store into a peer CTA's shared memory that completes transaction bytes on a barrier of that peer:
// data and signal travel together, no fence and no cluster-wide barrier on the sender side.
__device__ __forceinline__ void st_async_f32x2(uint32_t remote_addr, float a, float b, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               ::"r"(remote_addr), "f"(a), "f"(b), "r"(remote_bar)
               : "memory");
}

// ---- TMA ------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// smem -> global tile store (bulk async-group completion); OOB rows / columns are clipped by the tensor map
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(tmap), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
// smem tile += into global (element-wise fp32 add performed by the L2: no read of the destination by the SM)
__device__ __forceinline__ void tma_reduce_add_2d(const void* tmap, uint32_t src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(tmap), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_2d(const void* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, "
      "%7}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ---- thread-block clusters ----------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// shared::cluster address of `local_addr` (a shared::cta address) in CTA `cta_rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t local_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(cta_rank));
  return r;
}
// ---- wgmma (sm_90a warpgroup MMA) ------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// per-thread register limit of the executing warpgroup (all 128 threads execute it): producers hand registers to consumers
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// K-major, 128-byte-swizzled operand tile (rows of 64 bf16 = 128 B, 8-row atoms of 1024 B), as the TMA writes it with
// CU_TENSOR_MAP_SWIZZLE_128B: start address >> 4 | LBO (unused for swizzled K-major) = 1 | SBO = 1024 B | SWIZZLE_128B.
// Field layout of the sm_90 matrix descriptor (PTX ISA, "Matrix Descriptor Format" of wgmma).
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // [0,14)  start address
  d |= (uint64_t)1 << 16;                             // [16,30) leading byte offset (>>4)
  d |= (uint64_t)(1024 >> 4) << 32;                   // [32,46) stride byte offset (>>4)
  d |= (uint64_t)1 << 62;                             // [62,64) layout type SWIZZLE_128B
  return d;
}

// Same for 64-byte-swizzled tiles (rows of 32 bf16 = 64 B, 8-row atoms of 512 B, CU_TENSOR_MAP_SWIZZLE_64B): SBO = 512 B,
// layout type 2 = SWIZZLE_64B.  Tile starts are 512-byte aligned, so the base-offset field [49,52) stays 0.
__device__ __forceinline__ uint64_t make_sw64_kmajor_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // [0,14)  start address
  d |= (uint64_t)1 << 16;                             // [16,30) leading byte offset (>>4)
  d |= (uint64_t)(512 >> 4) << 32;                    // [32,46) stride byte offset (>>4)
  d |= (uint64_t)2 << 62;                             // [62,64) layout type SWIZZLE_64B
  return d;
}

}  // namespace ptx

// exact-erf GELU (torch nn.GELU() default), x * Phi(x), BRANCH-FREE and short:
//   Phi(x) = 1 - h (x >= 0) | h (x < 0),   h = 0.5 * erfc(|x| / sqrt 2)
//   erfc(z) = (a1 t + a2 t^2 + a3 t^3 + a4 t^4 + a5 t^5) * exp(-z^2),  t = 1 / (1 + p z)     (Abramowitz & Stegun 7.1.26,
//   |error| <= 1.5e-7), evaluated with one rcp.approx and one ex2.approx (MUFU pipe, otherwise idle in the epilogues) and
//   12 FMA-pipe instructions.  Max abs error of the GELU against the fp64 erf form over [-12, 12]: 4.2e-7
//   (tools/check_erf.py; torch's own fp32 GELU: 1.2e-6), and no cancellation for x < 0 (h is used directly).
// CUDA's erff() costs ~25 FMA-pipe instructions and takes a data-dependent branch; the fc1 epilogue of the split-bf16
// mode is FMA-pipe / issue bound (~30 instructions per element, from cycle counts of its warps), so the instruction count
// is what matters.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float p = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  p = fmaf(p, t, 0.5f * 1.421413741f);
  p = fmaf(p, t, 0.5f * -0.284496736f);
  p = fmaf(p, t, 0.5f * 0.254829592f);
  p *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * (z * -1.4426950408889634f)));
  const float h = p * e;
  return x * (x >= 0.0f ? 1.0f - h : h);
}

// ---- fp32 element pairs ----
// The FMA-pipe-bound epilogues and the depthwise convolution evaluate element PAIRS.  Each helper performs the same IEEE
// operation per lane (round-to-nearest, never contracted), so results do not depend on how the pair is issued.
typedef float2 f32x2_t;
__device__ __forceinline__ f32x2_t f2_pack(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ f32x2_t f2_dup(float v) { return make_float2(v, v); }
__device__ __forceinline__ float2 f2_unpack(f32x2_t v) { return v; }
__device__ __forceinline__ f32x2_t f2_fma(f32x2_t a, f32x2_t b, f32x2_t c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ f32x2_t f2_mul(f32x2_t a, f32x2_t b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2_t f2_add(f32x2_t a, f32x2_t b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2_t f2_sub(f32x2_t a, f32x2_t b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }

// gelu_erf for an element pair: the same A&S 7.1.26 evaluation without the selects (Phi = 0.5 + copysign(0.5 - h, x),
// the sign moved with one LOP3 per element on the ALU pipe) + 4 MUFU.
__device__ __forceinline__ f32x2_t gelu_erf2(f32x2_t x) {
  const float2 xf = f2_unpack(x);
  const f32x2_t z = f2_mul(x, f2_dup(0.70710678118654752440f));                 // signed; only z^2 and |z| are used
  const float2 zf = f2_unpack(z);
  const f32x2_t ta = f2_fma(f2_pack(fabsf(zf.x), fabsf(zf.y)), f2_dup(0.3275911f), f2_dup(1.0f));
  const float2 taf = f2_unpack(ta);
  float t0, t1;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(taf.x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(taf.y));
  const f32x2_t t = f2_pack(t0, t1);
  f32x2_t p = f2_fma(f2_dup(0.5f * 1.061405429f), t, f2_dup(0.5f * -1.453152027f));
  p = f2_fma(p, t, f2_dup(0.5f * 1.421413741f));
  p = f2_fma(p, t, f2_dup(0.5f * -0.284496736f));
  p = f2_fma(p, t, f2_dup(0.5f * 0.254829592f));
  p = f2_mul(p, t);
  const float2 ea = f2_unpack(f2_mul(f2_mul(z, z), f2_dup(-1.4426950408889634f)));
  float e0, e1;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(ea.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(ea.y));
  const float2 a = f2_unpack(f2_sub(f2_dup(0.5f), f2_mul(p, f2_pack(e0, e1))));   // 0.5 - h >= 0 (h <= 0.5)
  const float s0 = __uint_as_float(__float_as_uint(a.x) | (__float_as_uint(xf.x) & 0x80000000u));
  const float s1 = __uint_as_float(__float_as_uint(a.y) | (__float_as_uint(xf.y) & 0x80000000u));
  return f2_mul(x, f2_add(f2_pack(s0, s1), f2_dup(0.5f)));
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// GELU with packed half2 math (mode 1): 0.5*(1+tanh.approx.f16x2(x*(c0+c1*x^2))) evaluated for two
// elements per instruction, multiplied by the fp32 x.  ~5 instructions and 0.5 MUFU per element.
__device__ __forceinline__ uint32_t gelu_pack2_f16(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  const __half2 x2 = __hmul2(h, h);
  const __half2 pl = __hfma2(x2, __float2half2_rn(0.0356774f), __float2half2_rn(0.7978846f));
  const __half2 q = __hmul2(h, pl);
  uint32_t qi = *reinterpret_cast<const uint32_t*>(&q), ti;
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(ti) : "r"(qi));
  const __half2 t = *reinterpret_cast<const __half2*>(&ti);
  const __half2 phi = __hfma2(t, __float2half2_rn(0.5f), __float2half2_rn(0.5f));
  const float2 pf = __half22float2(phi);
  return pack_bf16(a * pf.x, b * pf.y);
}

// GELU for the GEMM epilogues: x * sigmoid(2*q(x)) with q an odd polynomial fitted so that
// 0.5*(1+tanh(q(x))) == Phi(x) (the erf form), evaluated with ex2.approx + rcp.approx
// (2 MUFU + 8 FMA-pipe instructions).  Coefficients: see tools/fit_gelu.py; max abs error vs the
// erf form is reported there and asserted in tests/test_gelu_fit.py.
#include "gelu_coeffs.h"
__device__ __forceinline__ float gelu_fast(float x) {
  float xc = fminf(fmaxf(x, -GELU_CLAMP), GELU_CLAMP);
  float x2 = xc * xc;
  float p = GELU_C3;
  p = fmaf(p, x2, GELU_C2);
  p = fmaf(p, x2, GELU_C1);
  p = fmaf(p, x2, GELU_C0);
  float e;  // exp2(-(2*log2e) * q)
  float t = xc * p;  // p already carries the -2*log2(e) factor
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}
#endif
