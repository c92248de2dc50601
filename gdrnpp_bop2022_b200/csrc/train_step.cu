// Parameter update of both trainers on the GPU: one Ranger step (GC + RAdam + lookahead) over every parameter of a
// model in one launch, and the model EMA in one launch.
//
// Replaces Ranger.step (lib/torch_utils/solver/ranger.py:102-202), about eleven torch ops per parameter tensor, and
// ModelEMA.update (det/yolox/utils/ema.py:50-60), two per state-dict entry.  DESIGN.md §7s pins every rule.  The host
// keeps what is naturally per-step host work (step counters, the radam_buffer cache, the fp32 scalars per tensor) and
// writes one GdrnRangerParam per tensor; the device walks (tensor, chunk) work units:
//   path 0  no GC: 8192-element chunks, element-wise.
//   path 1  GC, rows of at most 1024: each warp takes whole rows, stages the gradient row in shared memory, reduces
//           its mean in a fixed order and updates the row.
//   path 2  GC, rows of at most 8192: the CTA does the same for one row at a time.
//   path 3  GC, longer rows: 8192-element chunks; the row means come from rs_long_means_kernel, launched before.
// Every product and sum is rounded as the reference's torch ops round it on the GPU: the torch kernels evaluate
// `a + alpha * b` (add with alpha, addcmul, addcdiv) as one FMA, the rest as separately rounded operations.
#include "common.cuh"

static_assert(sizeof(GdrnRangerParam) == 128, "GdrnRangerParam is 128 bytes");
static_assert(sizeof(GdrnEmaEntry) == 32, "GdrnEmaEntry is 32 bytes");

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr long long RS_CHUNK = 8192;   // elements per unit
constexpr int RS_ROW_WARP = 1024;      // path 1 bound (one warp's shared-memory slice)
constexpr int RS_ROW_MAX = 8192;       // path 2 bound (the CTA's shared-memory row)
constexpr int RS_LONG_THREADS = 1024;
constexpr int RS_BATCH = 4;            // elements per thread in flight

enum { RF_GC = 1, RF_INIT = 2, RF_WD = 4, RF_ADAPTIVE = 8, RF_LOOKAHEAD = 16 };

struct Scal {
  float b1, c1, b2, c2, sl, wl, eps, alpha;
  int flags;
};

// smallest t with begin[t] + count[t] > u: the tensor that owns unit (or long row) u
template <typename F>
__device__ __forceinline__ int rs_find(int n, long long u, F end_of) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (end_of(mid) > u) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// one element: gradient g (centralised already), state at index i.  Writes p, m, v and slow.
__device__ __forceinline__ void rs_update(const Scal& s, float g, float* __restrict__ P, float* __restrict__ M,
                                          float* __restrict__ V, float* __restrict__ S, long long i, float p, float m,
                                          float v, float slow) {
  if (s.flags & RF_INIT) { m = 0.0f; v = 0.0f; slow = p; }
  v = __fmaf_rn(s.c2, __fmul_rn(g, g), __fmul_rn(v, s.b2));   // exp_avg_sq.mul_(b2).addcmul_(g, g, value=1-b2)
  m = __fmaf_rn(s.c1, g, __fmul_rn(m, s.b1));                  // exp_avg.mul_(b1).add_(g, alpha=1-b1)
  if (s.flags & RF_WD) p = __fmaf_rn(s.wl, p, p);              // p.add_(p, alpha=-wd*lr)
  if (s.flags & RF_ADAPTIVE) {
    const float denom = __fadd_rn(__fsqrt_rn(v), s.eps);       // exp_avg_sq.sqrt().add_(eps)
    p = __fmaf_rn(s.sl, __fdiv_rn(m, denom), p);               // p.addcdiv_(m, denom, value=-step_size*lr)
  } else {
    p = __fmaf_rn(s.sl, m, p);                                 // p.add_(m, alpha=-step_size*lr)
  }
  M[i] = m;
  V[i] = v;
  if (s.flags & RF_LOOKAHEAD) {
    slow = __fmaf_rn(s.alpha, __fsub_rn(p, slow), slow);      // slow.add_(p - slow, alpha=alpha)
    p = slow;
  }
  if (s.flags & (RF_LOOKAHEAD | RF_INIT)) S[i] = slow;
  P[i] = p;
}

// elements [first, first + len) of the tensor, thread `tid` of `nthr`, gradient from gsrc (shared memory, indexed
// from 0) or from global memory (gsrc == nullptr), minus `mean`; writes the centralised gradient back when GC is on.
__device__ __forceinline__ void rs_span(const GdrnRangerParam& d, const Scal& s, long long first, int len, int tid,
                                        int nthr, const float* gsrc, float mean, const float* __restrict__ long_means) {
  float* __restrict__ P = d.param;
  float* __restrict__ G = d.grad;
  float* __restrict__ M = d.exp_avg;
  float* __restrict__ V = d.exp_avg_sq;
  float* __restrict__ S = d.slow_buffer;
  const bool init = s.flags & RF_INIT, la = s.flags & RF_LOOKAHEAD, gc = s.flags & RF_GC;
  for (int j0 = tid; j0 < len; j0 += nthr * RS_BATCH) {
    float g[RS_BATCH], p[RS_BATCH], m[RS_BATCH], v[RS_BATCH], sl[RS_BATCH];
#pragma unroll
    for (int b = 0; b < RS_BATCH; ++b) {
      const int j = j0 + b * nthr;
      g[b] = p[b] = m[b] = v[b] = sl[b] = 0.0f;
      if (j < len) {
        const long long i = first + j;
        g[b] = gsrc ? gsrc[j] : G[i];
        p[b] = P[i];
        if (!init) { m[b] = M[i]; v[b] = V[i]; }
        if (la && !init) sl[b] = S[i];
      }
    }
#pragma unroll
    for (int b = 0; b < RS_BATCH; ++b) {
      const int j = j0 + b * nthr;
      if (j < len) {
        const long long i = first + j;
        float gg = g[b];
        if (gc) {
          const float mu = long_means ? long_means[d.mean_begin + i / d.row_len] : mean;
          gg = __fadd_rn(gg, -mu);                              // grad.add_(-(grad.mean(...)))
          G[i] = gg;
        }
        rs_update(s, gg, P, M, V, S, i, p[b], m[b], v[b], sl[b]);
      }
    }
  }
}

// fixed-order sum of one warp's doubles; every lane gets the same value (IEEE addition commutes)
__device__ __forceinline__ double rs_warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

__global__ void __launch_bounds__(RS_THREADS) rs_step_kernel(const GdrnRangerParam* __restrict__ T, int n,
                                                              const float* __restrict__ long_means) {
  __shared__ GdrnRangerParam d;
  __shared__ float srow[RS_ROW_MAX];
  __shared__ double sred[RS_WARPS];
  const long long u = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < (int)(sizeof(GdrnRangerParam) / 8)) {
    const int t = rs_find(n, u, [&](int k) { return T[k].unit_begin + T[k].units; });
    reinterpret_cast<long long*>(&d)[tid] = reinterpret_cast<const long long*>(T + t)[tid];
  }
  __syncthreads();
  const Scal s{d.beta1, d.one_minus_beta1, d.beta2, d.one_minus_beta2, d.neg_step_lr, d.neg_wd_lr, d.eps, d.alpha,
               d.flags};
  const long long k = u - d.unit_begin;
  if (d.path == 0 || d.path == 3) {
    const long long first = k * RS_CHUNK;
    const int len = (int)min(RS_CHUNK, d.numel - first);
    rs_span(d, s, first, len, tid, RS_THREADS, nullptr, 0.0f, d.path == 3 ? long_means : nullptr);
    return;
  }
  const long long L = d.row_len, rows = d.numel / L;
  const long long r0 = k * d.rows_per_unit, r1 = min(rows, r0 + d.rows_per_unit);
  if (d.path == 1) {   // one warp per row, the row in this warp's slice of srow
    float* gs = srow + warp * RS_ROW_WARP;
    for (long long r = r0 + warp; r < r1; r += RS_WARPS) {
      const float* gr = d.grad + r * L;
      double acc = 0.0;
      for (int j = lane; j < L; j += 32) {
        const float x = gr[j];
        gs[j] = x;
        acc += (double)x;
      }
      const float mean = (float)(rs_warp_sum(acc) / (double)L);
      __syncwarp();
      rs_span(d, s, r * L, (int)L, lane, 32, gs, mean, nullptr);
      __syncwarp();
    }
    return;
  }
  for (long long r = r0; r < r1; ++r) {   // path 2: the CTA per row
    const float* gr = d.grad + r * L;
    double acc = 0.0;
    for (int j = tid; j < L; j += RS_THREADS) {
      const float x = gr[j];
      srow[j] = x;
      acc += (double)x;
    }
    acc = rs_warp_sum(acc);
    if (lane == 0) sred[warp] = acc;
    __syncthreads();
    double tot = 0.0;
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) tot += sred[w];
    const float mean = (float)(tot / (double)L);
    rs_span(d, s, r * L, (int)L, tid, RS_THREADS, srow, mean, nullptr);
    __syncthreads();   // srow and sred are rewritten by the next row
  }
}

// one CTA per row longer than RS_ROW_MAX: its mean, summed in a fixed order in f64
__global__ void __launch_bounds__(RS_LONG_THREADS) rs_long_means_kernel(const GdrnRangerParam* __restrict__ T, int n,
                                                                        float* __restrict__ means) {
  __shared__ double sred[RS_LONG_THREADS / 32];
  const long long r = blockIdx.x;
  const int t = rs_find(n, r, [&](int k) {
    return T[k].mean_begin + (T[k].path == 3 ? T[k].numel / T[k].row_len : 0);
  });
  const long long L = T[t].row_len;
  const float* g = T[t].grad + (r - T[t].mean_begin) * L;
  double acc = 0.0;
  for (long long j = threadIdx.x; j < L; j += RS_LONG_THREADS) acc += (double)g[j];
  acc = rs_warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int w = 0; w < RS_LONG_THREADS / 32; ++w) tot += sred[w];
    means[r] = (float)(tot / (double)L);
  }
}

__global__ void __launch_bounds__(RS_THREADS) ema_kernel(const GdrnEmaEntry* __restrict__ E, int n, float dk,
                                                         float ck) {
  __shared__ GdrnEmaEntry e;
  const long long u = blockIdx.x;
  if (threadIdx.x < (int)(sizeof(GdrnEmaEntry) / 8)) {
    const int t = rs_find(n, u, [&](int k) {
      return E[k].unit_begin + (E[k].numel + RS_CHUNK - 1) / RS_CHUNK;
    });
    reinterpret_cast<long long*>(&e)[threadIdx.x] = reinterpret_cast<const long long*>(E + t)[threadIdx.x];
  }
  __syncthreads();
  const long long first = (u - e.unit_begin) * RS_CHUNK;
  const int len = (int)min(RS_CHUNK, e.numel - first);
  float* __restrict__ a = e.ema + first;
  const float* __restrict__ b = e.model + first;
  const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
  int j0 = 0;
  if (vec) {
    const int nv = len >> 2;
    for (int q = threadIdx.x; q < nv; q += RS_THREADS) {
      float4 x = reinterpret_cast<const float4*>(a)[q];
      const float4 y = reinterpret_cast<const float4*>(b)[q];
      x.x = __fadd_rn(__fmul_rn(x.x, dk), __fmul_rn(ck, y.x));   // v *= d; v += (1 - d) * m
      x.y = __fadd_rn(__fmul_rn(x.y, dk), __fmul_rn(ck, y.y));
      x.z = __fadd_rn(__fmul_rn(x.z, dk), __fmul_rn(ck, y.z));
      x.w = __fadd_rn(__fmul_rn(x.w, dk), __fmul_rn(ck, y.w));
      reinterpret_cast<float4*>(a)[q] = x;
    }
    j0 = nv << 2;
  }
  for (int j = j0 + threadIdx.x; j < len; j += RS_THREADS) a[j] = __fadd_rn(__fmul_rn(a[j], dk), __fmul_rn(ck, b[j]));
}

}  // namespace

extern "C" int gdrn_ranger_plan(GdrnRangerParam* params, int n, long long* n_units, long long* n_long_rows) {
  GDRN_REQUIRE(n >= 0 && (n == 0 || params) && n_units && n_long_rows, "gdrn_ranger_plan: bad arguments");
  long long units = 0, long_rows = 0;
  for (int t = 0; t < n; ++t) {
    GdrnRangerParam& d = params[t];
    GDRN_REQUIRE(d.numel >= 0, "gdrn_ranger_plan: negative numel");
    d.unit_begin = units;
    d.mean_begin = long_rows;
    d.rows_per_unit = 0;
    long long k = 0;
    if (d.numel == 0) {
      d.path = 0;
    } else if (!(d.flags & RF_GC)) {
      d.path = 0;
      k = (d.numel + RS_CHUNK - 1) / RS_CHUNK;
    } else {
      const long long L = d.row_len;
      GDRN_REQUIRE(L > 0 && d.numel % L == 0, "gdrn_ranger_plan: row_len does not divide numel");
      const long long rows = d.numel / L;
      if (L <= RS_ROW_MAX) {
        d.path = L <= RS_ROW_WARP ? 1 : 2;
        d.rows_per_unit = (int)(L <= RS_ROW_WARP ? max(RS_CHUNK / L, (long long)RS_WARPS) : max(RS_CHUNK / L, 1LL));
        k = (rows + d.rows_per_unit - 1) / d.rows_per_unit;
      } else {
        d.path = 3;
        long_rows += rows;
        k = (d.numel + RS_CHUNK - 1) / RS_CHUNK;
      }
    }
    GDRN_REQUIRE(k <= 0x7fffffff, "gdrn_ranger_plan: tensor too large");
    d.units = (int)k;
    units += k;
  }
  GDRN_REQUIRE(units <= 0x7fffffffLL && long_rows <= 0x7fffffffLL, "gdrn_ranger_plan: too many work units");
  *n_units = units;
  *n_long_rows = long_rows;
  return GDRN_OK;
}

extern "C" size_t gdrn_ranger_workspace_bytes(long long n_long_rows) {
  return n_long_rows > 0 ? (size_t)n_long_rows * sizeof(float) : 0;
}

extern "C" int gdrn_ranger_step(const GdrnRangerParam* params, int n, long long n_units, long long n_long_rows,
                                void* workspace, size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(n >= 0 && n_units >= 0 && n_long_rows >= 0 && n_units <= 0x7fffffffLL, "gdrn_ranger_step: bad sizes");
  if (n_units == 0) return GDRN_OK;
  GDRN_REQUIRE(params && n > 0, "gdrn_ranger_step: no parameter table");
  GDRN_REQUIRE(workspace_bytes >= gdrn_ranger_workspace_bytes(n_long_rows) && (n_long_rows == 0 || workspace),
               "gdrn_ranger_step: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float* means = n_long_rows ? (float*)workspace : nullptr;
  if (n_long_rows) {
    rs_long_means_kernel<<<(unsigned)n_long_rows, RS_LONG_THREADS, 0, st>>>(params, n, means);
    GDRN_CHECK_CUDA(cudaGetLastError());
    gdrn_count_launch(1);
  }
  rs_step_kernel<<<(unsigned)n_units, RS_THREADS, 0, st>>>(params, n, means);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}

extern "C" int gdrn_ema_plan(GdrnEmaEntry* entries, int n, long long* n_units) {
  GDRN_REQUIRE(n >= 0 && (n == 0 || entries) && n_units, "gdrn_ema_plan: bad arguments");
  long long units = 0;
  for (int t = 0; t < n; ++t) {
    GDRN_REQUIRE(entries[t].numel >= 0, "gdrn_ema_plan: negative numel");
    entries[t].unit_begin = units;
    units += (entries[t].numel + RS_CHUNK - 1) / RS_CHUNK;
  }
  GDRN_REQUIRE(units <= 0x7fffffffLL, "gdrn_ema_plan: too many work units");
  *n_units = units;
  return GDRN_OK;
}

extern "C" int gdrn_ema_update(const GdrnEmaEntry* entries, int n, long long n_units, float decay,
                               float one_minus_decay, void* stream) {
  GDRN_REQUIRE(n >= 0 && n_units >= 0 && n_units <= 0x7fffffffLL, "gdrn_ema_update: bad sizes");
  if (n_units == 0) return GDRN_OK;
  GDRN_REQUIRE(entries && n > 0, "gdrn_ema_update: no entry table");
  ema_kernel<<<(unsigned)n_units, RS_THREADS, 0, (cudaStream_t)stream>>>(entries, n, decay, one_minus_decay);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
