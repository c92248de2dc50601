// Error channel, version, and the exported plain-GEMM entry (tests + roofline measurement).
#include <stdlib.h>
#include <string.h>
#include <atomic>

#include <stdio.h>
#include <stdlib.h>
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
  uint64_t dims_a[2] = {(uint64_t)K, (uint64_t)M};
  uint64_t str_a[1] = {(uint64_t)K * 2};
  uint32_t box_a[2] = {64, 128};
  int rc = make_tmap_bf16(&p.tmap_a, A, 2, dims_a, str_a, box_a);
  if (rc) return rc;
  uint64_t dims_b[2] = {(uint64_t)K, (uint64_t)N};
  uint64_t str_b[1] = {(uint64_t)K * 2};
  uint32_t box_b[2] = {64, (uint32_t)block_n};
  rc = make_tmap_bf16(&p.tmap_b, W, 2, dims_b, str_b, box_b);
  if (rc) return rc;
  p.b_ptr = W; p.b_rows = N; p.b_ktot = K;
  p.a_rank = 2;
  p.num_taps = 1;
  p.k_chunks = (K + 63) / 64;
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
  static int trace_on = -1;
  if (trace_on < 0) trace_on = getenv("GDRN_GEMM_TRACE") ? 1 : 0;
  if (!trace_on) return gemm_tc_launch(p, block_n, (cudaStream_t)stream);
  // debug: cycle accounting of CTA 0, printed to stderr (synchronises the stream)
  static long long* d_trace = nullptr;
  if (!d_trace) GDRN_CHECK_CUDA(cudaMalloc(&d_trace, 16 * sizeof(long long)));
  GDRN_CHECK_CUDA(cudaMemsetAsync(d_trace, 0, 16 * sizeof(long long), (cudaStream_t)stream));
  p.trace = d_trace;
  rc = gemm_tc_launch(p, block_n, (cudaStream_t)stream);
  if (rc != GDRN_OK) return rc;
  long long h[16];
  GDRN_CHECK_CUDA(cudaMemcpyAsync(h, d_trace, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  GDRN_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  fprintf(stderr, "[gemm trace] M=%lld N=%d K=%d epi=%d bn=%d: cta0 cycles=%lld tiles=%lld | producer empty-wait=%lld | "
                  "consumer full-wait=%lld acc hand-over=%lld | epi0 acc-ld=%lld compute=%lld flush=%lld\n",
          (long long)M, N, K, epi, block_n, h[6], h[7], h[0], h[1], h[3], h[8], h[9], h[10]);
  return GDRN_OK;
}

extern "C" int gdrn_mlp_fused_x3(const void* A, const void* W1, const float* b1, const void* W2, const float* b2,
                                 const float* gamma, float* x, long long M, int C, void* stream) {
  GDRN_REQUIRE(A && W1 && b1 && W2 && b2 && gamma && x, "mlp_fused_x3: null argument");
  return mlp_fused_x3_launch(A, W1, b1, W2, b2, gamma, x, M, C, (cudaStream_t)stream);
}

extern "C" int gdrn_gemm_x3(const void* A, const void* W, const float* bias, const float* gamma, const float* resid,
                            void* out, int M, int N, int K, int epi, int block_n, void* stream);

extern "C" int gdrn_gemm_x3_ksplit(const void* A, const void* W, const float* bias, const float* gamma, float* x, int M, int N,
                                   int K, int block_n, unsigned* flags, int flag_words, void* stream) {
  GDRN_REQUIRE(flags != nullptr && flag_words > 0, "gemm_x3_ksplit: flags must be a zeroed device buffer");
  return gdrn_gemm_x3(A, W, bias, gamma, x, x, M, N, K, EPI_RESID, block_n, stream);
}

extern "C" int gdrn_gemm_x3(const void* A, const void* W, const float* bias, const float* gamma, const float* resid,
                            void* out, int M, int N, int K, int epi, int block_n, void* stream) {
  GDRN_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_x3: empty problem");
  GDRN_REQUIRE(K % 64 == 0, "gemm_x3: K must be a multiple of 64 (the lo half starts at a k-chunk boundary)");
  GDRN_REQUIRE(epi >= 0 && epi <= 2, "gemm_x3: epi must be 0 (store fp32), 1 (gelu -> split bf16) or 2 (resid)");
  GDRN_REQUIRE(block_n == 64 || block_n == 128 || block_n == 256, "gemm_x3: block_n must be 64, 128 or 256");
  GDRN_REQUIRE(N % 64 == 0, "gemm_x3: N must be a multiple of 64");
  GemmPlan p;
  memset(&p, 0, sizeof(p));
  uint64_t dims_a[2] = {(uint64_t)2 * K, (uint64_t)M};
  uint64_t str_a[1] = {(uint64_t)2 * K * 2};
  uint32_t box_a[2] = {64, 128};
  int rc = make_tmap_bf16(&p.tmap_a, A, 2, dims_a, str_a, box_a);
  if (rc) return rc;
  uint64_t dims_b[2] = {(uint64_t)2 * K, (uint64_t)N};
  uint64_t str_b[1] = {(uint64_t)2 * K * 2};
  uint32_t box_b[2] = {64, (uint32_t)block_n};
  rc = make_tmap_bf16(&p.tmap_b, W, 2, dims_b, str_b, box_b);
  if (rc) return rc;
  p.b_ptr = W; p.b_rows = N; p.b_ktot = 2LL * K;
  p.a_rank = 2;
  p.num_taps = 1;
  p.k_chunks = K / 64;
  p.taps[0] = {0, 0, 0, 0, 0};
  p.m_tiles = (M + 127) / 128;
  p.n_tiles = (N + block_n - 1) / block_n;
  p.M = M;
  p.N = N;
  p.epi = epi;
  p.out_f32 = epi == 1 ? 0 : 1;
  p.gelu_mode = 3;
  if (const char* e = getenv("GDRN_X3_GELU_MODE")) p.gelu_mode = atoi(e);   // 4 = libm erff (A/B experiments)
  p.split = 1; p.x3_a_lo = K; p.x3_b_lo = K;
  p.out = out;
  p.ldo = epi == 1 ? 2LL * N : N;
  p.bias = bias;
  p.gamma = gamma;
  p.resid = resid;
  static int trace_on = -1;
  if (trace_on < 0) trace_on = getenv("GDRN_GEMM_TRACE") ? 1 : 0;
  if (trace_on) {
    static long long* d_trace = nullptr;
    if (!d_trace) GDRN_CHECK_CUDA(cudaMalloc(&d_trace, 16 * sizeof(long long)));
    GDRN_CHECK_CUDA(cudaMemsetAsync(d_trace, 0, 16 * sizeof(long long), (cudaStream_t)stream));
    p.trace = d_trace;
    rc = gemm_tc_launch(p, block_n, (cudaStream_t)stream);
    if (rc != GDRN_OK) return rc;
    long long h[16];
    GDRN_CHECK_CUDA(cudaMemcpyAsync(h, d_trace, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    GDRN_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    fprintf(stderr, "[gemm x3 trace] M=%d N=%d K=%d epi=%d bn=%d: cta0 cycles=%lld tiles=%lld | producer empty-wait=%lld | "
                    "consumer full-wait=%lld acc hand-over=%lld | epi0 acc-ld=%lld compute=%lld flush=%lld\n",
            M, N, K, epi, block_n, h[6], h[7], h[0], h[1], h[3], h[8], h[9], h[10]);
    return GDRN_OK;
  }
  return gemm_tc_launch(p, block_n, (cudaStream_t)stream);
}

extern "C" int gdrn_dwconv_ln(const float* x, const float* w49c, const float* bias, const float* ln_w, const float* ln_b,
                              void* out, int B, int H, int W, int C, float eps, int split, int variant, void* stream) {
  GDRN_REQUIRE(x && w49c && bias && ln_w && ln_b && out, "dwconv_ln: null argument");
  GDRN_REQUIRE(variant >= -1 && variant <= 1, "dwconv_ln: variant must be -1 (default), 0 (per-tile cluster kernel) or 1 (ping-pong)");
  return launch_dwconv_ln_variant(x, w49c, bias, ln_w, ln_b, reinterpret_cast<__nv_bfloat16*>(out), B, H, W, C, eps, split, variant,
                                  (cudaStream_t)stream);
}
