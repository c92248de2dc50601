// Error channel, version, and the exported plain-GEMM entry (tests + roofline measurement).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>

#include "common.cuh"
#include "dense_ops.h"
#include "gemm_tc.h"

static thread_local char g_last_error[512] = "";

void gdrn_set_last_error(const char* file, int line, const char* msg) {
  const char* base = strrchr(file, '/');
  snprintf(g_last_error, sizeof(g_last_error), "%s:%d: %s", base ? base + 1 : file, line, msg);
}

static std::atomic<long long> g_launches{0};
void gdrn_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" long long gdrn_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

static std::atomic<uint64_t> g_gemm_kernels{0};
void gdrn_record_gemm_kernel(int id) { g_gemm_kernels.fetch_or(1ull << id, std::memory_order_relaxed); }
extern "C" uint64_t gdrn_gemm_kernels_launched(int reset) {
  return reset ? g_gemm_kernels.exchange(0, std::memory_order_relaxed) : g_gemm_kernels.load(std::memory_order_relaxed);
}

extern "C" const char* gdrn_last_error(void) { return g_last_error; }
extern "C" int gdrn_version(void) { return 100; }

extern "C" int gdrn_gemm_bf16(const void* A, const void* W, const float* bias, const float* gamma, const float* resid,
                              void* out, int M, int N, int K, int epi, int out_f32, int block_n, void* stream) {
  GDRN_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem");
  GDRN_REQUIRE(K % 8 == 0, "gemm: K must be a multiple of 8 (16-byte TMA row pitch)");
  GDRN_REQUIRE(epi >= 0 && epi <= 2, "gemm: epi must be 0 (store), 1 (gelu) or 2 (resid)");
  GDRN_REQUIRE(block_n < 64 || N % (block_n / 2 < 64 ? block_n / 2 : 64) == 0,
               "gemm: N must be a multiple of min(block_n/2, 64) for block_n >= 64");
  GemmPlan p;
  memset(&p, 0, sizeof(p));
  p.a_ptr = A; p.a_dims[0] = K; p.a_dims[1] = M; p.a_str[0] = (uint64_t)K * 2; p.a_box[1] = 128; p.a_k = K;
  p.b_ptr = W; p.b_rows = N; p.b_ktot = K;
  p.a_rank = 2;
  p.num_taps = 1;
  p.taps[0] = {0, 0, 0, 0, 0};
  p.m_tiles = (M + 127) / 128;
  p.n_tiles = (N + block_n - 1) / block_n;
  p.M = M;
  p.N = N;
  p.epi = epi;
  p.out_f32 = (epi == 2) ? 1 : (epi == 1 ? 0 : out_f32);
  if (const char* e = getenv("GDRN_GELU_MODE")) p.gelu_mode = atoi(e);
  p.out = out;
  p.ldo = N;
  p.bias = bias;
  p.gamma = gamma;
  p.resid = resid;
  return gemm_tc_launch(p, block_n, (cudaStream_t)stream);
}

extern "C" int gdrn_mlp_fused_x3(const void* A, const void* W1, const float* b1, const void* W2, const float* b2,
                                 const float* gamma, float* x, long long M, int C, void* stream) {
  GDRN_REQUIRE(A && W1 && b1 && W2 && b2 && gamma && x, "mlp_fused_x3: null argument");
  return mlp_fused_x3_launch(A, W1, b1, W2, b2, gamma, x, M, C, (cudaStream_t)stream);
}

extern "C" int gdrn_gemm_x3(const void* A, const void* W, const float* bias, const float* gamma, const float* resid,
                            void* out, int M, int N, int K, int epi, int block_n, void* stream) {
  GDRN_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_x3: empty problem");
  GDRN_REQUIRE(K % 64 == 0, "gemm_x3: K must be a multiple of 64 (the lo half starts at a k-chunk boundary)");
  GDRN_REQUIRE(epi >= 0 && epi <= 2, "gemm_x3: epi must be 0 (store fp32), 1 (gelu -> split bf16) or 2 (resid)");
  GDRN_REQUIRE(block_n == 64 || block_n == 128 || block_n == 256, "gemm_x3: block_n must be 64, 128 or 256");
  GDRN_REQUIRE(N % 64 == 0, "gemm_x3: N must be a multiple of 64");
  GDRN_REQUIRE(epi != 1 || (uintptr_t)out % 16 == 0,
               "gemm_x3: epi 1 needs a 16-byte aligned out (the split hi / lo rows leave through TMA stores)");
  GemmPlan p;
  memset(&p, 0, sizeof(p));
  p.a_ptr = A; p.a_dims[0] = 2ULL * K; p.a_dims[1] = M; p.a_str[0] = 4ULL * K; p.a_box[1] = 128; p.a_k = K;
  p.b_ptr = W; p.b_rows = N; p.b_ktot = 2LL * K;
  p.a_rank = 2;
  p.num_taps = 1;
  p.taps[0] = {0, 0, 0, 0, 0};
  p.m_tiles = (M + 127) / 128;
  p.n_tiles = (N + block_n - 1) / block_n;
  p.M = M;
  p.N = N;
  p.epi = epi;
  p.out_f32 = epi == 1 ? 0 : 1;
  p.gelu_mode = 3;
  p.split = 1; p.x3_a_lo = K; p.x3_b_lo = K;
  p.out = out;
  p.ldo = epi == 1 ? 2LL * N : N;
  p.bias = bias;
  p.gamma = gamma;
  p.resid = resid;
  return gemm_tc_launch(p, block_n, (cudaStream_t)stream);
}

extern "C" int gdrn_dwconv_ln(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                              void* out, int B, int H, int W, int C, float eps, int split, int variant, void* stream) {
  GDRN_REQUIRE(x && w49c && bias && ln_w && ln_b && out, "dwconv_ln: null argument");
  GDRN_REQUIRE(variant >= -1 && variant <= 1, "dwconv_ln: variant must be -1 (default), 0 (per-tile cluster kernel) or 1 (ping-pong)");
  return launch_dwconv_ln(x, w49c, bias, ln_w, ln_b, reinterpret_cast<__nv_bfloat16*>(out), B, H, W, C, eps, split, variant,
                          (cudaStream_t)stream);
}
