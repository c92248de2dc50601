// GdrnModel: weight repacking + forward orchestration of the dense path
// (GDRN_DoubleMask.forward, eval branch: core/gdrn_modeling/models/GDRN_double_mask.py:96-214).
//
// Data layout in HBM (per forward of `B` ROIs; all activations NHWC):
//   X     fp32  [B,h,w,C]    residual stream of the current ConvNeXt stage (updated in place by fc2's epilogue)
//   A     bf16  [M,K]        GEMM A operand produced by the CUDA-core front halves (dwconv+LN, LN+patchify, stem)
//   Hb    bf16  [M,4C]       fc1 output (GELU applied in the GEMM epilogue)
//   feat  bf16  [B,8,8,C3]   backbone output
//   R     bf16  [B,64,64,256] raw conv output of the geometry head (pre-GroupNorm) + GN statistics (double)
//   P,Q   bf16  [B,64,64,256] post GN+GELU(+bilinear) activations (ping-pong)
//   pnp_in bf16 [B,64,64,128] Patch-PnP input assembled by the out-conv epilogue
// Weights: bf16 [N][taps*K] K-major per GEMM, fp32 vectors for bias / gamma / norm affine.
//
// Precision 1 ("bf16x3", split-bf16): every bf16 GEMM operand v is stored as the pair hi = bf16(v), lo = bf16(v - hi)
// -- activations as rows [hi C | lo C], weights as rows [hi Ktot | lo Ktot] -- and every GEMM accumulates the three
// products A_lo*W_hi + A_hi*W_lo + A_hi*W_hi in the same fp32 accumulator (operand error 2^-17 instead of
// 2^-9).  Head conv outputs stay fp32 until GroupNorm, GELU is the exact erf form, and the Patch-PnP FC stack runs
// in fp32 on the CUDA cores.  Used to meet the 1e-4 rad / 1e-3 parity bar of BASELINE.json against the fp32 oracle.
#include <algorithm>
#include <map>
#include <string>
#include <vector>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "dense_ops.h"
#include "gemm_tc.h"

namespace {

struct Arch {
  int depths[4];
  int dims[4];   // channels of the reference model
  int cp[4];     // stored channel width: dims rounded up to a multiple of 64 (GEMM k-chunk / depthwise channel slice); the pad
                 // channels carry zero weights, biases and affines everywhere, so they stay exactly zero through the network
};

bool get_arch(const char* name, Arch* a) {
  if (!strcmp(name, "convnext_base")) *a = {{3, 3, 27, 3}, {128, 256, 512, 1024}, {0, 0, 0, 0}};
  else if (!strcmp(name, "convnext_small")) *a = {{3, 3, 27, 3}, {96, 192, 384, 768}, {0, 0, 0, 0}};
  else if (!strcmp(name, "convnext_tiny")) *a = {{3, 3, 9, 3}, {96, 192, 384, 768}, {0, 0, 0, 0}};
  else return false;
  for (int s = 0; s < 4; ++s) a->cp[s] = (a->dims[s] + 63) / 64 * 64;
  return true;
}

struct BlockW {
  float* dw_w;   // [49][C]
  float* dw_b;   // [C]
  float* ln_w; float* ln_b;
  __nv_bfloat16* fc1_w;  // [4C][C]
  float* fc1_b;
  __nv_bfloat16* fc2_w;  // [C][4C]
  float* fc2_b;
  float* gamma;
};

struct LoadOp {  // one repack of a source tensor into a destination buffer
  void* dst;
  int dst_is_bf16;
  PackDesc d;
  long long expect_numel;
};

}  // namespace

struct GdrnModel {
  Arch arch;
  int num_classes;
  int max_batch;
  int in_res = 256, out_res = 64;
  int fuse_mlp = 1;   // fused fc1->GELU->fc2 kernel where supported (env GDRN_MLP_FUSED=0 disables)
  int fuse_mlp_x3 = 1;  // the same in split-bf16 mode, stage 0 (env GDRN_MLP_FUSED_X3=0 disables)
  int precise = 0;    // 0: bf16 operands (fast); 1: split-bf16 x3 products, fp32 FC stack, erf GELU
  int gelu_mode = 1;  // fc1 epilogue GELU: 1 = packed-half2 tanh.approx (default, fastest), 0 = fp32 ex2/rcp form, 2 = fp32 tanh.approx; env GDRN_GELU_MODE
  // ---- weights (device) ----
  std::vector<void*> allocs;
  __nv_bfloat16* stem_w;  // [C0][64]
  float *stem_b, *stem_ln_w, *stem_ln_b;
  struct Down { float *ln_w, *ln_b; __nv_bfloat16* w; float* b; } down[4];
  std::vector<BlockW> blocks[4];
  // head
  __nv_bfloat16* deconv_w[4];  // per output parity (py*2+px): [256][ntaps*C3]
  float *gn_w[7], *gn_b[7];    // features.1, 3.gn, 4.gn, 6.gn, 7.gn, 9.gn, 10.gn
  __nv_bfloat16* hconv_w[6];   // features.{3,4,6,7,9,10}.conv : [256][9*256]
  __nv_bfloat16* out_w;        // [num_classes][80][256]
  float* out_b;                // [num_classes][80]
  // pnp
  __nv_bfloat16* pconv_w[3];   // [128][9*128]
  float *pgn_w[3], *pgn_b[3];
  __nv_bfloat16* pfc1_w;       // [1024][8192] (columns permuted to NHWC flatten order)
  float* pfc1_b;
  __nv_bfloat16* pfc2_w;       // [256][1024]
  float* pfc2_b;
  __nv_bfloat16* pfcrt_w;      // [16][256]: rows 0-5 fc_r, 6-8 fc_t, rest 0
  float* pfcrt_b;              // [16]
  float *pfc1_wf = nullptr, *pfc2_wf = nullptr, *pfcrt_wf = nullptr;  // precise mode: fp32 copies (same layouts)
  // ---- loader ----
  std::map<std::string, std::vector<LoadOp>> loaders;
  std::map<std::string, bool> loaded;
  int missing = 0;
  // ---- optional per-category timing (bench.py roofline) ----
  bool prof_on = false;
  std::vector<cudaEvent_t> prof_events;
  std::vector<int> prof_cat;
  int prof_used = 0;
};

namespace {

template <typename T>
T* dalloc(GdrnModel* m, size_t n, bool zero = true) {
  void* p = nullptr;
  if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) return nullptr;
  if (zero) cudaMemset(p, 0, n * sizeof(T));
  m->allocs.push_back(p);
  return reinterpret_cast<T*>(p);
}

void add_loader(GdrnModel* m, const std::string& key, void* dst, int is_bf16, PackDesc d, long long numel) {
  LoadOp op;
  op.dst = dst;
  op.dst_is_bf16 = is_bf16;
  op.d = d;
  op.expect_numel = numel;
  if (m->loaders.find(key) == m->loaders.end()) {
    m->loaded[key] = false;
    m->missing++;
  }
  m->loaders[key].push_back(op);
}

PackDesc pd(long long d0, long long d1, long long d2, long long d3, long long s0, long long s1, long long s2,
            long long s3, long long t0, long long t1, long long t2, long long t3, long long soff = 0,
            long long doff = 0, long long lo = 0) {
  PackDesc d;
  d.dims[0] = d0; d.dims[1] = d1; d.dims[2] = d2; d.dims[3] = d3;
  d.ss[0] = s0; d.ss[1] = s1; d.ss[2] = s2; d.ss[3] = s3;
  d.ds[0] = t0; d.ds[1] = t1; d.ds[2] = t2; d.ds[3] = t3;
  d.soff = soff; d.doff = doff; d.lo_delta = lo;
  return d;
}

// plain copy of a vector / matrix [r][c] -> [r][ldc]
void add_copy(GdrnModel* m, const std::string& key, void* dst, int is_bf16, long long rows, long long cols,
              long long ld_dst, long long doff = 0, long long lo = 0) {
  add_loader(m, key, dst, is_bf16, pd(1, 1, rows, cols, 0, 0, cols, 1, 0, 0, ld_dst, 1, 0, doff, lo), rows * cols);
}

bool build_weights(GdrnModel* m) {
  const Arch& a = m->arch;
  const int C0 = a.dims[0], C0p = a.cp[0], C3 = a.dims[3], C3p = a.cp[3];
  const int nc = m->num_classes;
  const int S = m->precise ? 2 : 1;  // bf16 weight rows are [hi Ktot | lo Ktot] in precise mode
  auto LO = [&](long long ktot) { return S == 2 ? ktot : 0LL; };
  bool ok = true;
#define ALLOC(ptr, T, n) ok = ok && ((ptr = dalloc<T>(m, (n))) != nullptr)
  // ---- stem ----
  ALLOC(m->stem_w, __nv_bfloat16, (size_t)S * C0p * 64);
  ALLOC(m->stem_b, float, C0p); ALLOC(m->stem_ln_w, float, C0p); ALLOC(m->stem_ln_b, float, C0p);
  if (!ok) return false;
  add_copy(m, "backbone.stem_0.weight", m->stem_w, 1, C0, 48, S * 64, 0, LO(64));
  add_copy(m, "backbone.stem_0.bias", m->stem_b, 0, 1, C0, C0);
  add_copy(m, "backbone.stem_1.weight", m->stem_ln_w, 0, 1, C0, C0);
  add_copy(m, "backbone.stem_1.bias", m->stem_ln_b, 0, 1, C0, C0);
  for (int s = 0; s < 4; ++s) {
    const int C = a.dims[s], Cp = a.cp[s];
    char buf[160];
    if (s > 0) {
      const int Ci = a.dims[s - 1], Cip = a.cp[s - 1];
      ALLOC(m->down[s].ln_w, float, Cip); ALLOC(m->down[s].ln_b, float, Cip);
      ALLOC(m->down[s].w, __nv_bfloat16, (size_t)S * Cp * 4 * Cip);
      ALLOC(m->down[s].b, float, Cp);
      if (!ok) return false;
      snprintf(buf, sizeof(buf), "backbone.stages_%d.downsample.0.weight", s); add_copy(m, buf, m->down[s].ln_w, 0, 1, Ci, Ci);
      snprintf(buf, sizeof(buf), "backbone.stages_%d.downsample.0.bias", s); add_copy(m, buf, m->down[s].ln_b, 0, 1, Ci, Ci);
      // [C][Ci][2][2] -> [C][tap][Ci]
      snprintf(buf, sizeof(buf), "backbone.stages_%d.downsample.1.weight", s);
      add_loader(m, buf, m->down[s].w, 1, pd(1, C, 4, Ci, 0, (long long)Ci * 4, 1, 4, 0, (long long)S * 4 * Cip, Cip, 1, 0, 0, LO(4 * Cip)), (long long)C * Ci * 4);
      snprintf(buf, sizeof(buf), "backbone.stages_%d.downsample.1.bias", s); add_copy(m, buf, m->down[s].b, 0, 1, C, C);
    }
    m->blocks[s].resize(a.depths[s]);
    for (int i = 0; i < a.depths[s]; ++i) {
      BlockW& w = m->blocks[s][i];
      ALLOC(w.dw_w, float, (size_t)49 * Cp); ALLOC(w.dw_b, float, Cp); ALLOC(w.ln_w, float, Cp); ALLOC(w.ln_b, float, Cp);
      ALLOC(w.fc1_w, __nv_bfloat16, (size_t)S * 4 * C * Cp); ALLOC(w.fc1_b, float, 4 * C);   // hidden width stays 4 * C
      ALLOC(w.fc2_w, __nv_bfloat16, (size_t)S * 4 * C * Cp); ALLOC(w.fc2_b, float, Cp); ALLOC(w.gamma, float, Cp);
      if (!ok) return false;
      std::string p = "backbone.stages_" + std::to_string(s) + ".blocks." + std::to_string(i) + ".";
      // conv_dw.weight [C][1][7][7] -> [49][C]
      add_loader(m, p + "conv_dw.weight", w.dw_w, 0, pd(1, 1, 49, C, 0, 0, 1, 49, 0, 0, Cp, 1), (long long)C * 49);
      add_copy(m, p + "conv_dw.bias", w.dw_b, 0, 1, C, C);
      add_copy(m, p + "norm.weight", w.ln_w, 0, 1, C, C);
      add_copy(m, p + "norm.bias", w.ln_b, 0, 1, C, C);
      add_copy(m, p + "mlp.fc1.weight", w.fc1_w, 1, 4 * C, C, S * Cp, 0, LO(Cp));
      add_copy(m, p + "mlp.fc1.bias", w.fc1_b, 0, 1, 4 * C, 4 * C);
      add_copy(m, p + "mlp.fc2.weight", w.fc2_w, 1, C, 4 * C, S * 4 * C, 0, LO(4 * C));
      add_copy(m, p + "mlp.fc2.bias", w.fc2_b, 0, 1, C, C);
      add_copy(m, p + "gamma", w.gamma, 0, 1, C, C);
    }
  }
  // ---- geometry head ----
  // ConvTranspose2d weight [C3][256][3][3]; out(2a+py, 2b+px) taps: py=0 -> ky=1 (iy=a); py=1 -> ky=0 (iy=a+1), ky=2 (iy=a)
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      const int nty = py ? 2 : 1, ntx = px ? 2 : 1;
      const int par = py * 2 + px;
      ALLOC(m->deconv_w[par], __nv_bfloat16, (size_t)S * 256 * nty * ntx * C3p);
      if (!ok) return false;
      // dst [o][jy][jx][i]; src index = i*256*9 + o*9 + (ky*3+kx), ky = py ? 2*jy : 1, kx = px ? 2*jx : 1
      const long long soff = (py ? 0 : 3) + (px ? 0 : 1);
      // dims (o, jy, jx, i)
      PackDesc d = pd(256, nty, ntx, C3, 9, 6, 2, (long long)256 * 9, (long long)S * nty * ntx * C3p, (long long)ntx * C3p, C3p, 1, soff, 0,
                      LO((long long)nty * ntx * C3p));
      add_loader(m, "geo_head_net.features.0.weight", m->deconv_w[par], 1, d, (long long)C3 * 256 * 9);
    }
  const char* gn_names[7] = {"features.1", "features.3.gn", "features.4.gn", "features.6.gn",
                             "features.7.gn", "features.9.gn", "features.10.gn"};
  for (int i = 0; i < 7; ++i) {
    ALLOC(m->gn_w[i], float, 256); ALLOC(m->gn_b[i], float, 256);
    if (!ok) return false;
    add_copy(m, std::string("geo_head_net.") + gn_names[i] + ".weight", m->gn_w[i], 0, 1, 256, 256);
    add_copy(m, std::string("geo_head_net.") + gn_names[i] + ".bias", m->gn_b[i], 0, 1, 256, 256);
  }
  const int conv_ids[6] = {3, 4, 6, 7, 9, 10};
  for (int i = 0; i < 6; ++i) {
    ALLOC(m->hconv_w[i], __nv_bfloat16, (size_t)S * 256 * 9 * 256);
    if (!ok) return false;
    // [O][I][3][3] -> [O][tap][I]
    add_loader(m, "geo_head_net.features." + std::to_string(conv_ids[i]) + ".conv.weight", m->hconv_w[i], 1,
               pd(1, 256, 9, 256, 0, 256 * 9, 1, 9, 0, S * 9 * 256, 256, 1, 0, 0, LO(9 * 256)), 256LL * 256 * 9);
  }
  // out layer: [nc*70][256] -> gathered [nc][80][256], rows: vis c | full nc+c | x 2nc+c | y 3nc+c | z 4nc+c | region 5nc+65c+j
  ALLOC(m->out_w, __nv_bfloat16, (size_t)S * nc * 80 * 256);
  ALLOC(m->out_b, float, (size_t)nc * 80);
  if (!ok) return false;
  add_loader(m, "geo_head_net.out_layer.weight", m->out_w, 1,
             pd(1, nc, 5, 256, 0, 256, (long long)nc * 256, 1, 0, S * 80 * 256, S * 256, 1, 0, 0, LO(256)), (long long)nc * 70 * 256);
  add_loader(m, "geo_head_net.out_layer.weight", m->out_w, 1,
             pd(1, nc, 65, 256, 0, 65 * 256, 256, 1, 0, S * 80 * 256, S * 256, 1, (long long)5 * nc * 256, S * 5 * 256, LO(256)),
             (long long)nc * 70 * 256);
  add_loader(m, "geo_head_net.out_layer.bias", m->out_b, 0, pd(1, 1, nc, 5, 0, 0, 1, nc, 0, 0, 80, 1), (long long)nc * 70);
  add_loader(m, "geo_head_net.out_layer.bias", m->out_b, 0, pd(1, 1, nc, 65, 0, 0, 65, 1, 0, 0, 80, 1, 5LL * nc, 5),
             (long long)nc * 70);
  // ---- Patch-PnP ----
  for (int i = 0; i < 3; ++i) {
    const int cin = i == 0 ? 69 : 128;
    ALLOC(m->pconv_w[i], __nv_bfloat16, (size_t)S * 128 * 9 * 128);
    ALLOC(m->pgn_w[i], float, 128); ALLOC(m->pgn_b[i], float, 128);
    if (!ok) return false;
    add_loader(m, "pnp_net.features." + std::to_string(i * 3) + ".weight", m->pconv_w[i], 1,
               pd(1, 128, 9, cin, 0, (long long)cin * 9, 1, 9, 0, S * 9 * 128, 128, 1, 0, 0, LO(9 * 128)), 128LL * cin * 9);
    add_copy(m, "pnp_net.features." + std::to_string(i * 3 + 1) + ".weight", m->pgn_w[i], 0, 1, 128, 128);
    add_copy(m, "pnp_net.features." + std::to_string(i * 3 + 1) + ".bias", m->pgn_b[i], 0, 1, 128, 128);
  }
  ALLOC(m->pfc1_w, __nv_bfloat16, (size_t)1024 * 8192); ALLOC(m->pfc1_b, float, 1024);
  ALLOC(m->pfc2_w, __nv_bfloat16, (size_t)256 * 1024); ALLOC(m->pfc2_b, float, 256);
  ALLOC(m->pfcrt_w, __nv_bfloat16, (size_t)16 * 256); ALLOC(m->pfcrt_b, float, 16);
  if (!ok) return false;
  // fc1 [1024][c*64 + hw] -> [1024][hw*128 + c]
  add_loader(m, "pnp_net.fc1.weight", m->pfc1_w, 1, pd(1, 1024, 64, 128, 0, 8192, 1, 64, 0, 8192, 128, 1), 1024LL * 8192);
  add_copy(m, "pnp_net.fc1.bias", m->pfc1_b, 0, 1, 1024, 1024);
  add_copy(m, "pnp_net.fc2.weight", m->pfc2_w, 1, 256, 1024, 1024);
  add_copy(m, "pnp_net.fc2.bias", m->pfc2_b, 0, 1, 256, 256);
  add_copy(m, "pnp_net.fc_r.weight", m->pfcrt_w, 1, 6, 256, 256, 0);
  add_copy(m, "pnp_net.fc_t.weight", m->pfcrt_w, 1, 3, 256, 256, 6 * 256);
  add_copy(m, "pnp_net.fc_r.bias", m->pfcrt_b, 0, 1, 6, 6, 0);
  add_copy(m, "pnp_net.fc_t.bias", m->pfcrt_b, 0, 1, 3, 3, 6);
  if (m->precise) {  // fp32 FC stack
    ALLOC(m->pfc1_wf, float, (size_t)1024 * 8192); ALLOC(m->pfc2_wf, float, (size_t)256 * 1024);
    ALLOC(m->pfcrt_wf, float, (size_t)16 * 256);
    if (!ok) return false;
    add_loader(m, "pnp_net.fc1.weight", m->pfc1_wf, 0, pd(1, 1024, 64, 128, 0, 8192, 1, 64, 0, 8192, 128, 1), 1024LL * 8192);
    add_copy(m, "pnp_net.fc2.weight", m->pfc2_wf, 0, 256, 1024, 1024);
    add_copy(m, "pnp_net.fc_r.weight", m->pfcrt_wf, 0, 6, 256, 256, 0);
    add_copy(m, "pnp_net.fc_t.weight", m->pfcrt_wf, 0, 3, 256, 256, 6 * 256);
  }
#undef ALLOC
  return ok;
}

// ---- workspace carving ----
struct Workspace {
  float* X;
  __nv_bfloat16* A;
  __nv_bfloat16* Hb;
  __nv_bfloat16* feat;
  __nv_bfloat16 *R, *P, *Q;
  __nv_bfloat16* pnp_in;
  __nv_bfloat16 *pR, *pP;
  __nv_bfloat16 *f1, *f2;
  float *pF, *f1f, *f2f;  // precise mode: fp32 Patch-PnP feature [B,8192] and FC activations
  float* fc_part;         // precise mode: K-slice partial sums of the fp32 FC stack
  float* fout;      // [B][16]
  double* gn_stats; // [10][B][32][2]
  size_t zero_bytes;    // gn_stats: cleared at the start of every forward
  float* gn_mr;     // [B][32][2] mean / rstd scratch of the layer being applied
  size_t total;
};

size_t align_up(size_t v) { return (v + 1023) & ~(size_t)1023; }

Workspace carve(const GdrnModel* m, int B, void* base) {
  const Arch& a = m->arch;
  Workspace w;
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* r = p ? p + off : nullptr; off += align_up(bytes); return r; };
  const size_t M0 = (size_t)B * 64 * 64;
  const size_t S = m->precise ? 2 : 1;  // split-bf16 rows are twice as wide
  size_t x_el = 0, a_el = M0 * 64, h_el = 0;
  for (int s = 0; s < 4; ++s) {
    size_t Ms = M0 >> (2 * s);
    x_el = std::max(x_el, Ms * a.cp[s]);
    a_el = std::max(a_el, Ms * a.cp[s]);
    h_el = std::max(h_el, Ms * a.dims[s] * 4);
  }
  w.X = reinterpret_cast<float*>(take(x_el * 4));
  w.A = reinterpret_cast<__nv_bfloat16*>(take(S * a_el * 2));
  w.Hb = reinterpret_cast<__nv_bfloat16*>(take(S * h_el * 2));
  w.feat = reinterpret_cast<__nv_bfloat16*>(take(S * B * 64 * a.cp[3] * 2));
  w.R = reinterpret_cast<__nv_bfloat16*>(take(S * M0 * 256 * 2));  // precise: fp32 [M0,256]
  w.P = reinterpret_cast<__nv_bfloat16*>(take(S * M0 * 256 * 2));
  w.Q = reinterpret_cast<__nv_bfloat16*>(take(S * M0 * 256 * 2));
  w.pnp_in = reinterpret_cast<__nv_bfloat16*>(take(S * M0 * 128 * 2));
  w.pR = reinterpret_cast<__nv_bfloat16*>(take(S * B * 32 * 32 * 128 * 2));  // precise: fp32
  w.pP = reinterpret_cast<__nv_bfloat16*>(take(S * B * 32 * 32 * 128 * 2));
  w.pF = reinterpret_cast<float*>(take(m->precise ? (size_t)B * 8192 * 4 : 0));
  w.f1f = reinterpret_cast<float*>(take(m->precise ? (size_t)B * 1024 * 4 : 0));
  w.f2f = reinterpret_cast<float*>(take(m->precise ? (size_t)B * 256 * 4 : 0));
  w.fc_part = reinterpret_cast<float*>(take(m->precise ? fc_f32_part_bytes(B, 1024) : 0));
  w.f1 = reinterpret_cast<__nv_bfloat16*>(take((size_t)B * 1024 * 2));
  w.f2 = reinterpret_cast<__nv_bfloat16*>(take((size_t)B * 256 * 2));
  w.fout = reinterpret_cast<float*>(take((size_t)B * 16 * 4));
  w.gn_stats = reinterpret_cast<double*>(take((size_t)10 * B * 32 * 2 * 8));
  w.zero_bytes = (size_t)10 * B * 32 * 2 * 8;
  w.gn_mr = reinterpret_cast<float*>(take((size_t)B * 32 * 2 * 4));
  w.total = off;
  return w;
}

int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

// A = plain [M,K] rows
// S = 2: rows are [hi K | lo K] (split-bf16); the tap list is expanded by expand_x3() afterwards
// A operand geometry; gemm_tc_launch encodes the tensor map with the k-chunk width of the kernel it picks
void set_a(GemmPlan& p, const void* A, int rank, const uint64_t* dims, const uint64_t* str, const uint32_t* box, int K) {
  p.a_rank = rank;
  p.a_ptr = A;
  for (int i = 0; i < rank; ++i) {
    p.a_dims[i] = dims[i];
    p.a_box[i] = box[i];
    if (i > 0) p.a_str[i - 1] = str[i - 1];
  }
  p.a_k = K;
}

int plan_a2d(GemmPlan& p, const void* A, long long M, int K, int S = 1) {
  uint64_t dims[2] = {(uint64_t)S * K, (uint64_t)M};
  uint64_t str[1] = {(uint64_t)S * K * 2};
  uint32_t box[2] = {0, 128};
  set_a(p, A, 2, dims, str, box, K);
  p.num_taps = 1;
  p.taps[0] = {0, 0, 0, 0, 0};
  p.m_tiles = (int)((M + 127) / 128);
  p.M = (int)M;
  return GDRN_OK;
}

int plan_b(GemmPlan& p, const void* W, long long rows, long long Ktot, int block_n, int N, int S = 1) {
  p.N = N;
  p.n_tiles = (N + block_n - 1) / block_n;
  p.b_ptr = W; p.b_rows = rows; p.b_ktot = (long long)S * Ktot;
  return GDRN_OK;
}

// A = NHWC [B,H,W,C] pixel boxes; output grid OHxOW = (H*osy, W*osx) handled by the caller's mapping fields
int plan_a4d(GemmPlan& p, const void* act, int B, int H, int W, int C, int S = 1) {
  int bw = W >= 128 ? 128 : W;
  int bh = 128 / bw; if (bh > H) bh = H;
  int bb = 128 / (bw * bh);
  const uint64_t RC_ = (uint64_t)S * C;  // row (pixel) width in elements
  uint64_t dims[4] = {RC_, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  uint64_t str[3] = {RC_ * 2, (uint64_t)W * RC_ * 2, (uint64_t)H * W * RC_ * 2};
  uint32_t box[4] = {0, (uint32_t)bw, (uint32_t)bh, (uint32_t)bb};
  set_a(p, act, 4, dims, str, box, C);
  p.lg_bw = ilog2(bw); p.lg_bh = ilog2(bh); p.lg_bb = ilog2(bb);
  p.tiles_x = W / bw; p.tiles_y = H / bh;
  p.m_tiles = p.tiles_x * p.tiles_y * ((B + bb - 1) / bb);
  p.M = B;
  return GDRN_OK;
}

// stride-2 view of NHWC [B,H,W,C]: (2C, W/2, 2, H/2, B); output grid (H/2 x W/2)
int plan_a5d_s2(GemmPlan& p, const void* act, int B, int H, int W, int C, int S = 1) {
  const int OW = W / 2, OH = H / 2;
  int bw = OW >= 128 ? 128 : OW;
  int bh = 128 / bw; if (bh > OH) bh = OH;
  int bb = 128 / (bw * bh);
  const uint64_t RC_ = (uint64_t)S * C;
  uint64_t dims[5] = {2 * RC_, (uint64_t)OW, 2, (uint64_t)OH, (uint64_t)B};
  uint64_t str[4] = {2 * RC_ * 2, (uint64_t)W * RC_ * 2, (uint64_t)2 * W * RC_ * 2, (uint64_t)H * W * RC_ * 2};
  uint32_t box[5] = {0, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bb};
  set_a(p, act, 5, dims, str, box, C);
  p.lg_bw = ilog2(bw); p.lg_bh = ilog2(bh); p.lg_bb = ilog2(bb);
  p.tiles_x = OW / bw; p.tiles_y = OH / bh;
  p.m_tiles = p.tiles_x * p.tiles_y * ((B + bb - 1) / bb);
  p.M = B;
  return GDRN_OK;
}

// split-bf16: taps[] keeps listing the hi operands; gemm_tc_launch expands them to the three products
void set_x3(GemmPlan& p, int a_lo_c0, int b_lo_off) {
  p.split = 1;
  p.x3_a_lo = a_lo_c0;
  p.x3_b_lo = b_lo_off;
}

#define RC(expr) do { int _rc = (expr); if (_rc != GDRN_OK) return _rc; } while (0)
// profiled launch: category 0 = wgmma GEMM, 1 = depthwise conv + LN, 2 = other CUDA-core kernels
#define RCP(cat, expr) do { prof_begin(m, (cat), st); int _rc = (expr); prof_end(m, st); if (_rc != GDRN_OK) return _rc; } while (0)

void prof_begin(GdrnModel* m, int cat, cudaStream_t st) {
  if (!m->prof_on) return;
  if (m->prof_used + 2 > (int)m->prof_events.size()) {
    for (int i = 0; i < 64; ++i) { cudaEvent_t e; cudaEventCreate(&e); m->prof_events.push_back(e); }
  }
  m->prof_cat.push_back(cat);
  cudaEventRecord(m->prof_events[m->prof_used], st);
}
void prof_end(GdrnModel* m, cudaStream_t st) {
  if (!m->prof_on) return;
  cudaEventRecord(m->prof_events[m->prof_used + 1], st);
  m->prof_used += 2;
}

// tile width: the largest one the N dimension divides into (the CTA-pair kernels need N % block_n == 0) that still yields
// at least half a wave of CTAs; small batches (the per-image case: 5 ROIs, BASELINE configs[4]) otherwise run their long-K
// GEMMs on a dozen SMs (stage-2 fc2 at B = 5: 20 CTAs of 96 k-iterations, 51 us -> 80 CTAs at width 64)
int pick_bn(int N, long long M) {
  const int half_wave = gdrn_num_sms() / 2;
  const long long m_tiles = (M + 127) / 128;
  int bn = N % 256 == 0 ? 256 : (N % 128 == 0 ? 128 : 64);
  while (bn > 64 && m_tiles * (N / bn) < half_wave) bn >>= 1;
  return bn;
}

void reset_plan(GemmPlan& p) { memset(&p, 0, sizeof(p)); }

// run_stage names: true when `name` is `prefix` followed by a decimal index (and, with j, "_" and a second one); no sign,
// no leading zeros
bool stage_index(const char* name, const char* prefix, int* i, int* j = nullptr) {
  const size_t l = strlen(prefix);
  if (strncmp(name, prefix, l)) return false;
  const char* p = name + l;
  auto number = [&p](int* v) {
    if (*p < '0' || *p > '9' || (p[0] == '0' && p[1] >= '0' && p[1] <= '9')) return false;
    int x = 0;
    for (int n = 0; *p >= '0' && *p <= '9'; ++n, ++p) {
      if (n == 6) return false;
      x = 10 * x + (*p - '0');
    }
    *v = x;
    return true;
  };
  if (!number(i)) return false;
  if (j && (*p++ != '_' || !number(j))) return false;
  return *p == 0;
}

// GroupNorm sums of head layer i (0: deconv, 1..6: head convs, 7..9: Patch-PnP convs)
double* stat_slot(const Workspace& w, int B, int i) { return w.gn_stats + (size_t)i * B * 32 * 2; }

// ---------------- ConvNeXt backbone, one function per stage ----------------
// The residual stream lives in w.X (fp32 NHWC, stored width cp[s]); each stage updates it in place.  gdrn_model_forward
// runs them in order; gdrn_model_run_stage runs one of them on its own.

// stem: roi_img [B,3,256,256] -> 4x4/s4 conv as GEMM (K=48 padded to 64) + bias + LayerNorm2d in the epilogue -> w.X [B,64,64,cp0]
int stage_stem(GdrnModel* m, const Workspace& w, int B, const float* roi_img, cudaStream_t st) {
  const int PR = m->precise, S = PR ? 2 : 1;
  const int C0 = m->arch.dims[0], C0p = m->arch.cp[0];
  const long long M0 = (long long)B * 64 * 64;
  RCP(2, launch_stem_patchify(roi_img, w.A, B, 256, 256, PR, st));
  if (C0p != 128) {   // convnext_base (128) and tiny / small (96 stored 128 wide: pad rows of stem_w are zero)
    gdrn_set_last_error(__FILE__, __LINE__, "forward: the fused stem epilogue needs a 128-wide (padded) first stage");
    return GDRN_ERR_INVALID;
  }
  GemmPlan p;
  reset_plan(p);
  RC(plan_a2d(p, w.A, M0, 64, S));
  RC(plan_b(p, m->stem_w, C0p, 64, 128, C0p, S));
  if (PR) set_x3(p, 64, 64);
  p.epi = EPI_BIAS_LN; p.out = w.X; p.ldo = C0p; p.bias = m->stem_b;
  p.ln_w = m->stem_ln_w; p.ln_b = m->stem_ln_b; p.ln_eps = 1e-6f; p.ln_n = C0;
  RCP(0, gemm_tc_launch(p, 128, st));
  return GDRN_OK;
}

// downsample in front of stage s (1..3): LayerNorm2d + 2x2 patchify of w.X [B,2r,2r,cp[s-1]] into the operand w.A
// [B*r*r, 4*cp[s-1]], then the 2x2/s2 conv as GEMM + bias into w.X [B,r,r,cp[s]], r = 64 >> s
int stage_downsample(GdrnModel* m, const Workspace& w, int B, int s, cudaStream_t st) {
  const Arch& a = m->arch;
  const int PR = m->precise, S = PR ? 2 : 1;
  const int C = a.cp[s], Ci = a.cp[s - 1];
  const int res = 64 >> s;
  RCP(2, launch_ln_patchify2(w.X, m->down[s].ln_w, m->down[s].ln_b, w.A, B, 2 * res, 2 * res, Ci, 1e-6f, PR, st, a.dims[s - 1]));
  const long long M = (long long)B * res * res;
  GemmPlan p;
  reset_plan(p);
  RC(plan_a2d(p, w.A, M, 4 * Ci, S));
  const int bn = pick_bn(C, M);
  RC(plan_b(p, m->down[s].w, C, 4 * Ci, bn, C, S));
  if (PR) set_x3(p, 4 * Ci, 4 * Ci);
  p.epi = EPI_STORE; p.out_f32 = 1; p.out = w.X; p.ldo = C; p.bias = m->down[s].b;
  RCP(0, gemm_tc_launch(p, bn, st));
  return GDRN_OK;
}

// block i of stage s on w.X [B,r,r,cp[s]], r = 64 >> s: depthwise 7x7 + LayerNorm into the operand w.A [B*r*r, cp[s]], then
// the MLP fc1 -> GELU -> fc2 -> *gamma -> +residual back into w.X (one fused kernel where supported, else two GEMMs via w.Hb)
int stage_block(GdrnModel* m, const Workspace& w, int B, int s, int i, cudaStream_t st) {
  const Arch& a = m->arch;
  const int PR = m->precise, S = PR ? 2 : 1;
  const int gelu_mode = PR ? 3 : m->gelu_mode;
  const int res = 64 >> s;
  const int Cr = a.dims[s];   // channels of the reference model
  const int C = a.cp[s];      // stored width (pad channels are zero)
  const int H4 = 4 * Cr;      // hidden width of the MLP
  const long long M = (long long)B * res * res;
  const BlockW& bw = m->blocks[s][i];
  RCP(1, launch_dwconv_ln(w.X, bw.dw_w, bw.dw_b, bw.ln_w, bw.ln_b, w.A, B, res, res, C, 1e-6f, PR, -1, st, Cr));
  if (!PR && m->fuse_mlp && m->gelu_mode == 1 && Cr == C && mlp_fused_supported(C, M)) {
    // stage 0: fc1 -> GELU -> fc2 -> residual in one kernel (no 4C-wide Hb round trip through HBM)
    RCP(0, mlp_fused_launch(w.A, bw.fc1_w, bw.fc1_b, bw.fc2_w, bw.fc2_b, bw.gamma, w.X, M, C, st));
    return GDRN_OK;
  }
  if (PR && m->fuse_mlp_x3 && Cr == C && mlp_fused_x3_supported(C, M)) {
    RCP(0, mlp_fused_x3_launch(w.A, bw.fc1_w, bw.fc1_b, bw.fc2_w, bw.fc2_b, bw.gamma, w.X, M, C, st));
    return GDRN_OK;
  }
  GemmPlan p;
  reset_plan(p);
  RC(plan_a2d(p, w.A, M, C, S));
  const int bn1 = pick_bn(H4, M);
  RC(plan_b(p, bw.fc1_w, H4, C, bn1, H4, S));
  if (PR) set_x3(p, C, C);
  p.epi = EPI_GELU; p.gelu_mode = gelu_mode; p.out = w.Hb; p.ldo = S * H4; p.bias = bw.fc1_b;
  RCP(0, gemm_tc_launch(p, bn1, st));
  reset_plan(p);
  RC(plan_a2d(p, w.Hb, M, H4, S));
  const int bn2 = pick_bn(C, M);
  RC(plan_b(p, bw.fc2_w, C, H4, bn2, C, S));
  if (PR) set_x3(p, H4, H4);
  p.epi = EPI_RESID; p.out_f32 = 1; p.out = w.X; p.resid = w.X; p.ldo = C; p.bias = bw.fc2_b; p.gamma = bw.gamma;
  RCP(0, gemm_tc_launch(p, bn2, st));
  return GDRN_OK;
}

// ---------------- geometry head and Patch-PnP, one function per stage ----------------
// gdrn_model_forward runs them in this order; gdrn_model_run_stage runs one of them on its own.

// deconv 3x3 s2 (8x8 -> 16x16) as four parity GEMMs into w.R + GN + GELU into `out` [B,16,16,256]
int stage_deconv(GdrnModel* m, const Workspace& w, int B, const __nv_bfloat16* feat, __nv_bfloat16* out, cudaStream_t st) {
  const int PR = m->precise, S = PR ? 2 : 1;
  const int C3 = m->arch.cp[3];
  GemmPlan p;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      reset_plan(p);
      RC(plan_a4d(p, feat, B, 8, 8, C3, S));
      int nt = 0;
      for (int jy = 0; jy < (py ? 2 : 1); ++jy)
        for (int jx = 0; jx < (px ? 2 : 1); ++jx) {
          // ky = py ? 2*jy : 1 -> iy = a + (ky == 0 ? 1 : 0)
          const int dy = (py && jy == 0) ? 1 : 0, dx = (px && jx == 0) ? 1 : 0;
          p.taps[nt] = {0, dx, dy, 0, nt * C3};
          ++nt;
        }
      p.num_taps = nt;
      // only B/2 row tiles (8x8 inputs): narrow N tiles so that the launch still covers the SMs
      const int dbn = p.m_tiles >= 96 ? 256 : 64;
      RC(plan_b(p, m->deconv_w[py * 2 + px], 256, (long long)nt * C3, dbn, 256, S));
      if (PR) set_x3(p, C3, nt * C3);
      p.epi = EPI_GNSTATS; p.out_f32 = PR; p.out = w.R; p.ldo = 256;
      p.OH = 16; p.OW = 16; p.osy = 2; p.osx = 2; p.ooy = py; p.oox = px;
      p.gn_stats = stat_slot(w, B, 0); p.gn_groups = 32; p.gn_cpg = 8;
      RCP(0, gemm_tc_launch(p, dbn, st));
    }
  RCP(2, launch_gn_gelu(w.R, PR, stat_slot(w, B, 0), w.gn_mr, m->gn_w[0], m->gn_b[0], out, B, 16, 16, 256, 32, 1e-5f, PR, st));
  return GDRN_OK;
}

// head conv li (0..5, at 16, 16, 32, 32, 64, 64 pixels): 3x3 conv into w.R + GN + GELU into `out`; after convs 1 and 3 the
// GN + GELU result goes to `in` (the conv's input, dead by then) and the bilinear x2 of it to `out`
int stage_head_conv(GdrnModel* m, const Workspace& w, int B, int li, __nv_bfloat16* in, __nv_bfloat16* out, cudaStream_t st) {
  const int PR = m->precise, S = PR ? 2 : 1;
  const int hres = 16 << (li / 2);
  GemmPlan p;
  reset_plan(p);
  RC(plan_a4d(p, in, B, hres, hres, 256, S));
  for (int t = 0; t < 9; ++t) p.taps[t] = {0, t % 3 - 1, t / 3 - 1, 0, t * 256};
  p.num_taps = 9;
  const int hbn = pick_bn(256, (long long)B * hres * hres);   // narrower tiles when a small batch leaves most SMs without one
  RC(plan_b(p, m->hconv_w[li], 256, 9 * 256, hbn, 256, S));
  if (PR) set_x3(p, 256, 9 * 256);
  p.epi = EPI_GNSTATS; p.out_f32 = PR; p.out = w.R; p.ldo = 256;
  p.OH = hres; p.OW = hres; p.osy = 1; p.osx = 1; p.ooy = 0; p.oox = 0;
  p.gn_stats = stat_slot(w, B, li + 1); p.gn_groups = 32; p.gn_cpg = 8;
  RCP(0, gemm_tc_launch(p, hbn, st));
  if (li % 2 == 0 || li == 5) {
    RCP(2, launch_gn_gelu(w.R, PR, stat_slot(w, B, li + 1), w.gn_mr, m->gn_w[li + 1], m->gn_b[li + 1], out, B, hres, hres, 256, 32,
                          1e-5f, PR, st));
  } else {
    RCP(2, launch_gn_gelu(w.R, PR, stat_slot(w, B, li + 1), w.gn_mr, m->gn_w[li + 1], m->gn_b[li + 1], in, B, hres, hres, 256, 32,
                          1e-5f, PR, st));
    RCP(2, launch_upsample2x(in, out, B, hres, hres, 256, PR, st));
  }
  return GDRN_OK;
}

// out conv (class gathered) + Patch-PnP input assembly into w.pnp_in (+ the optional NCHW maps)
int stage_out_conv(GdrnModel* m, const Workspace& w, int B, const __nv_bfloat16* in, const int64_t* roi_classes,
                   const float* roi_extents, const float* roi_coord_2d, const GdrnMaps* maps, cudaStream_t st) {
  const int PR = m->precise, S = PR ? 2 : 1;
  GemmPlan p;
  reset_plan(p);
  RC(plan_a2d(p, in, (long long)B * 64 * 64, 256, S));
  RC(plan_b(p, m->out_w, (long long)m->num_classes * 80, 256, 80, 80, S));
  if (PR) set_x3(p, 256, 256);
  p.n_tiles = 1;
  p.b_rows_per_class = 80;
  p.epi = EPI_OUTCONV;
  p.roi_classes = reinterpret_cast<const long long*>(roi_classes);
  p.num_classes = m->num_classes;
  p.rows_per_roi = 4096;
  p.oc_bias = m->out_b;
  p.roi_extents = roi_extents;
  p.roi_coord_2d = roi_coord_2d;
  p.pnp_in = w.pnp_in;
  if (maps && maps->mask) {
    GDRN_REQUIRE(maps->full_mask && maps->coor_x && maps->coor_y && maps->coor_z && maps->region,
                 "forward: GdrnMaps must be all set or all NULL");
    p.map_mask = maps->mask; p.map_full = maps->full_mask; p.map_x = maps->coor_x; p.map_y = maps->coor_y;
    p.map_z = maps->coor_z; p.map_region = maps->region;
  }
  RCP(0, gemm_tc_launch(p, 80, st));
  return GDRN_OK;
}

// Patch-PnP conv i (0..2): 3x3 s2 conv of `in` [B,2r,2r,128] into w.pR + GN + GELU into w.pP [B,r,r,128] (split-bf16 mode,
// i = 2: fp32 into w.pF, the input of the fp32 FC stack)
int stage_pnp_conv(GdrnModel* m, const Workspace& w, int B, int i, const __nv_bfloat16* in, cudaStream_t st) {
  const int PR = m->precise, S = PR ? 2 : 1;
  const int ires = 64 >> i, ores = ires / 2;
  GemmPlan p;
  reset_plan(p);
  RC(plan_a5d_s2(p, in, B, ires, ires, 128, S));
  // input (2*o + k - 1): k=0 -> parity 1, half index o-1; k=1 -> parity 0, o; k=2 -> parity 1, o
  for (int t = 0; t < 9; ++t) {
    const int ky = t / 3, kx = t % 3;
    const int pyy = (ky == 1) ? 0 : 1, dyy = (ky == 0) ? -1 : 0;
    const int pxx = (kx == 1) ? 0 : 1, dxx = (kx == 0) ? -1 : 0;
    p.taps[t] = {pxx * S * 128, dxx, pyy, dyy, t * 128};
  }
  p.num_taps = 9;
  RC(plan_b(p, m->pconv_w[i], 128, 9 * 128, 128, 128, S));
  if (PR) set_x3(p, 128, 9 * 128);
  p.epi = EPI_GNSTATS; p.out_f32 = PR; p.out = w.pR; p.ldo = 128;
  p.OH = ores; p.OW = ores; p.osy = 1; p.osx = 1;
  p.gn_stats = stat_slot(w, B, 7 + i); p.gn_groups = 32; p.gn_cpg = 4;
  RCP(0, gemm_tc_launch(p, 128, st));
  if (PR && i == 2) {  // last feature map feeds the fp32 FC stack
    RCP(2, launch_gn_gelu_f32(reinterpret_cast<const float*>(w.pR), stat_slot(w, B, 7 + i), w.gn_mr, m->pgn_w[i], m->pgn_b[i], w.pF, B,
                              ores, ores, 128, 32, 1e-5f, st));
  } else {
    // the conv has read its input (pnp_in or pP) by now: GN + GELU may overwrite pP
    RCP(2, launch_gn_gelu(w.pR, PR, stat_slot(w, B, 7 + i), w.gn_mr, m->pgn_w[i], m->pgn_b[i], w.pP, B, ores, ores, 128, 32, 1e-5f, PR, st));
  }
  return GDRN_OK;
}

// FC stack: Patch-PnP feature [B,8192] (w.pF fp32 in split-bf16 mode, w.pP bf16 otherwise) -> 1024 -> 256 -> 9 into w.fout [B,16]
int stage_pnp_fc(GdrnModel* m, const Workspace& w, int B, cudaStream_t st) {
  if (m->precise) {
    RCP(2, launch_fc_f32(w.pF, m->pfc1_wf, m->pfc1_b, w.f1f, w.fc_part, B, 1024, 8192, 1024, 1, st));
    RCP(2, launch_fc_f32(w.f1f, m->pfc2_wf, m->pfc2_b, w.f2f, w.fc_part, B, 256, 1024, 256, 1, st));
    RCP(2, launch_fc_f32(w.f2f, m->pfcrt_wf, m->pfcrt_b, w.fout, w.fc_part, B, 16, 256, 16, 0, st));
    return GDRN_OK;
  }
  GemmPlan p;
  reset_plan(p);
  RC(plan_a2d(p, w.pP, B, 8192));
  RC(plan_b(p, m->pfc1_w, 1024, 8192, 64, 1024));
  p.epi = EPI_GELU; p.gelu_mode = 0; p.out = w.f1; p.ldo = 1024; p.bias = m->pfc1_b;
  RCP(0, gemm_tc_launch(p, 64, st));
  reset_plan(p);
  RC(plan_a2d(p, w.f1, B, 1024));
  RC(plan_b(p, m->pfc2_w, 256, 1024, 64, 256));
  p.epi = EPI_GELU; p.gelu_mode = 0; p.out = w.f2; p.ldo = 256; p.bias = m->pfc2_b;
  RCP(0, gemm_tc_launch(p, 64, st));
  reset_plan(p);
  RC(plan_a2d(p, w.f2, B, 256));
  RC(plan_b(p, m->pfcrt_w, 16, 256, 16, 16));
  p.epi = EPI_STORE; p.out_f32 = 1; p.out = w.fout; p.ldo = 16; p.bias = m->pfcrt_b;
  RCP(0, gemm_tc_launch(p, 16, st));
  return GDRN_OK;
}

}  // namespace

// ================================================================================================
extern "C" int gdrn_model_create(GdrnModel** out, const char* arch, int num_classes, int max_batch) {
  int precision = 1;  // split-bf16 (fp32 parity) unless GDRN_PRECISION=0 asks for the bf16 throughput mode
  if (const char* e = getenv("GDRN_PRECISION")) precision = atoi(e);
  return gdrn_model_create_ex(out, arch, num_classes, max_batch, precision);
}

extern "C" int gdrn_model_precision(const GdrnModel* m) { return m ? m->precise : -1; }

extern "C" int gdrn_model_create_ex(GdrnModel** out, const char* arch, int num_classes, int max_batch, int precision) {
  GDRN_REQUIRE(out != nullptr && arch != nullptr, "model_create: null argument");
  GDRN_REQUIRE(precision == 0 || precision == 1, "model_create: precision must be 0 (bf16) or 1 (split-bf16 x3)");
  Arch a;
  GDRN_REQUIRE(get_arch(arch, &a), "model_create: unknown arch (convnext_base | convnext_small | convnext_tiny)");
  GDRN_REQUIRE(num_classes >= 1 && num_classes <= 64 && max_batch >= 1, "model_create: bad num_classes / max_batch");
  GdrnModel* m = new GdrnModel();
  m->arch = a;
  m->num_classes = num_classes;
  m->max_batch = max_batch;
  m->precise = precision;
  if (const char* e = getenv("GDRN_GELU_MODE")) m->gelu_mode = atoi(e);
  if (const char* e = getenv("GDRN_MLP_FUSED")) m->fuse_mlp = atoi(e);
  if (const char* e = getenv("GDRN_MLP_FUSED_X3")) m->fuse_mlp_x3 = atoi(e);
  if (!build_weights(m)) {
    gdrn_model_destroy(m);
    gdrn_set_last_error(__FILE__, __LINE__, "model_create: cudaMalloc failed");
    return GDRN_ERR_CUDA;
  }
  *out = m;
  return GDRN_OK;
}

extern "C" void gdrn_model_destroy(GdrnModel* m) {
  if (!m) return;
  for (void* p : m->allocs) cudaFree(p);
  for (cudaEvent_t e : m->prof_events) cudaEventDestroy(e);
  delete m;
}

extern "C" int gdrn_model_load_tensor(GdrnModel* m, const char* key, const float* data, int64_t numel, void* stream) {
  GDRN_REQUIRE(m && key && data, "load_tensor: null argument");
  auto it = m->loaders.find(key);
  if (it == m->loaders.end()) {
    char msg[256];
    snprintf(msg, sizeof(msg), "load_tensor: unknown key '%s'", key);
    gdrn_set_last_error(__FILE__, __LINE__, msg);
    return GDRN_ERR_INVALID;
  }
  for (const LoadOp& op : it->second) {
    if (op.expect_numel != numel) {
      char msg[256];
      snprintf(msg, sizeof(msg), "load_tensor: '%s' has %lld elements, expected %lld", key, (long long)numel,
               op.expect_numel);
      gdrn_set_last_error(__FILE__, __LINE__, msg);
      return GDRN_ERR_INVALID;
    }
    RC(launch_pack(data, op.dst, op.dst_is_bf16, op.d, (cudaStream_t)stream));
  }
  if (!m->loaded[key]) {
    m->loaded[key] = true;
    m->missing--;
  }
  return GDRN_OK;
}

extern "C" int gdrn_model_missing(const GdrnModel* m) { return m ? m->missing : -1; }

extern "C" size_t gdrn_model_workspace_bytes(const GdrnModel* m, int batch) {
  if (!m || batch < 1) return 0;
  return carve(m, batch, nullptr).total + 1024;
}

extern "C" int gdrn_model_forward(GdrnModel* m, const float* roi_img, const int64_t* roi_classes,
                                  const float* roi_coord_2d, const float* roi_cams, const float* roi_centers,
                                  const float* roi_whs, const float* resize_ratios, const float* roi_extents, int batch,
                                  float* out_rot, float* out_trans, float* out_raw, const GdrnMaps* maps,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  GDRN_REQUIRE(m != nullptr, "forward: null model");
  if (m->missing != 0) {
    gdrn_set_last_error(__FILE__, __LINE__, "forward: model weights not fully loaded");
    return GDRN_ERR_STATE;
  }
  GDRN_REQUIRE(batch >= 1 && batch <= m->max_batch, "forward: batch out of range");
  GDRN_REQUIRE(roi_img && roi_coord_2d && roi_cams && roi_centers && roi_whs && resize_ratios &&
                   roi_extents && out_rot && out_trans && workspace,
               "forward: null argument");
  // a class-agnostic head (one class slab) reads no labels; a class-aware one needs them
  GDRN_REQUIRE(roi_classes || m->num_classes == 1, "forward: roi_classes is NULL but the head is class-aware");
  const size_t need = gdrn_model_workspace_bytes(m, batch);
  if (workspace_bytes < need) {
    gdrn_set_last_error(__FILE__, __LINE__, "forward: workspace too small");
    return GDRN_ERR_STATE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int B = batch;
  const Arch& a = m->arch;
  void* wbase = reinterpret_cast<void*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~(uintptr_t)1023);
  Workspace w = carve(m, B, wbase);
  m->prof_used = 0;
  m->prof_cat.clear();
  GDRN_CHECK_CUDA(cudaMemsetAsync(w.gn_stats, 0, w.zero_bytes, st));   // GroupNorm sums

  const int PR = m->precise;

  // ---------------- ConvNeXt backbone ----------------
  RC(stage_stem(m, w, B, roi_img, st));
  for (int s = 0; s < 4; ++s) {
    if (s > 0) RC(stage_downsample(m, w, B, s, st));
    for (int i = 0; i < a.depths[s]; ++i) RC(stage_block(m, w, B, s, i, st));
  }
  const int C3 = a.cp[3];
  if (PR) RCP(2, launch_cast_split(w.X, w.feat, (long long)B * 64, C3, st));
  else RCP(2, launch_cast_bf16(w.X, w.feat, (long long)B * 64 * C3, st));

  // ---------------- geometry head ----------------
  RC(stage_deconv(m, w, B, w.feat, w.P, st));
  __nv_bfloat16* cur = w.P;
  __nv_bfloat16* nxt = w.Q;
  for (int li = 0; li < 6; ++li) {
    RC(stage_head_conv(m, w, B, li, cur, nxt, st));
    std::swap(cur, nxt);
  }
  RC(stage_out_conv(m, w, B, cur, roi_classes, roi_extents, roi_coord_2d, maps, st));

  // ---------------- Patch-PnP ----------------
  for (int i = 0; i < 3; ++i) RC(stage_pnp_conv(m, w, B, i, i == 0 ? w.pnp_in : w.pP, st));
  RC(stage_pnp_fc(m, w, B, st));
  RCP(2, launch_pose_lift(w.fout, 16, roi_cams, roi_centers, roi_whs, resize_ratios, out_rot, out_trans, out_raw, B, st));
  return GDRN_OK;
}

extern "C" int gdrn_model_set_profiling(GdrnModel* m, int enable) {
  GDRN_REQUIRE(m != nullptr, "set_profiling: null model");
  m->prof_on = enable != 0;
  return GDRN_OK;
}

// Sums the CUDA-event durations of the last forward per category (blocks until that forward finished).
extern "C" int gdrn_model_get_profile(GdrnModel* m, float* ms_out /*[3]*/, int* launches_out /*[3]*/) {
  GDRN_REQUIRE(m && ms_out && launches_out, "get_profile: null argument");
  for (int c = 0; c < 3; ++c) { ms_out[c] = 0.f; launches_out[c] = 0; }
  if (m->prof_used == 0) return GDRN_OK;
  GDRN_CHECK_CUDA(cudaEventSynchronize(m->prof_events[m->prof_used - 1]));
  for (int i = 0; i < m->prof_used / 2; ++i) {
    float ms = 0.f;
    GDRN_CHECK_CUDA(cudaEventElapsedTime(&ms, m->prof_events[2 * i], m->prof_events[2 * i + 1]));
    const int c = m->prof_cat[i];
    ms_out[c] += ms;
    launches_out[c] += 1;
  }
  return GDRN_OK;
}

extern "C" int64_t gdrn_model_debug_read(GdrnModel* m, const char* name, int batch, float* dst, void* workspace,
                                         void* stream) {
  if (!m || !name || !dst || !workspace) return GDRN_ERR_INVALID;
  void* wbase = reinterpret_cast<void*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~(uintptr_t)1023);
  Workspace w = carve(m, batch, wbase);
  cudaStream_t st = (cudaStream_t)stream;
  const int C3 = m->arch.dims[3];
  long long n = 0;
  if (m->precise && strcmp(name, "stage3_x") && strcmp(name, "fc_out")) {
    gdrn_set_last_error(__FILE__, __LINE__, "debug_read: only stage3_x / fc_out are readable in split-bf16 mode");
    return GDRN_ERR_INVALID;
  }
  if (!strcmp(name, "conv_feat")) {
    n = (long long)batch * 64 * C3;
    if (launch_bf16_to_f32(w.feat, dst, n, st)) return GDRN_ERR_CUDA;
  } else if (!strcmp(name, "stage3_x")) {
    n = (long long)batch * 64 * C3;
    if (cudaMemcpyAsync(dst, w.X, n * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return GDRN_ERR_CUDA;
  } else if (!strcmp(name, "pnp_in")) {
    n = (long long)batch * 4096 * 128;
    if (launch_bf16_to_f32(w.pnp_in, dst, n, st)) return GDRN_ERR_CUDA;
  } else if (!strcmp(name, "pnp_feat")) {
    n = (long long)batch * 8192;
    if (launch_bf16_to_f32(w.pP, dst, n, st)) return GDRN_ERR_CUDA;
  } else if (!strcmp(name, "head64")) {
    // after 6 swaps starting from cur=P: cur == P again
    n = (long long)batch * 4096 * 256;
    if (launch_bf16_to_f32(w.P, dst, n, st)) return GDRN_ERR_CUDA;
  } else if (!strcmp(name, "fc_out")) {
    n = (long long)batch * 16;
    if (cudaMemcpyAsync(dst, w.fout, n * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return GDRN_ERR_CUDA;
  } else {
    gdrn_set_last_error(__FILE__, __LINE__, "debug_read: unknown name");
    return GDRN_ERR_INVALID;
  }
  return n;
}

extern "C" int gdrn_model_run_stage(GdrnModel* m, const char* stage, int batch, const float* in, float* out, float* raw_out,
                                    double* gn_stats_out, const int64_t* roi_classes, const float* roi_extents,
                                    const float* roi_coord_2d, const GdrnMaps* maps, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  GDRN_REQUIRE(m && stage && in && out && workspace, "run_stage: null argument");
  if (m->missing != 0) {
    gdrn_set_last_error(__FILE__, __LINE__, "run_stage: model weights not fully loaded");
    return GDRN_ERR_STATE;
  }
  GDRN_REQUIRE(batch >= 1 && batch <= m->max_batch, "run_stage: batch out of range");
  if (workspace_bytes < gdrn_model_workspace_bytes(m, batch)) {
    gdrn_set_last_error(__FILE__, __LINE__, "run_stage: workspace too small");
    return GDRN_ERR_STATE;
  }
  const Arch& a = m->arch;
  // indexed stages: "head_conv<i>", "pnp_conv<i>", "down<s>", "block<s>_<i>"
  int li = -1, pi = -1, ds = -1, bs = -1, bi = -1;
  const bool stem = !strcmp(stage, "stem");
  const bool down = stage_index(stage, "down", &ds), block = stage_index(stage, "block", &bs, &bi);
  const bool head_conv = stage_index(stage, "head_conv", &li), pnp_conv = stage_index(stage, "pnp_conv", &pi);
  const bool deconv = !strcmp(stage, "deconv"), out_conv = !strcmp(stage, "out_conv"), pnp_fc = !strcmp(stage, "pnp_fc");
  GDRN_REQUIRE(stem || down || block || deconv || head_conv || out_conv || pnp_conv || pnp_fc, "run_stage: unknown stage");
  GDRN_REQUIRE(!head_conv || li < 6, "run_stage: head_conv index out of range (0..5)");
  GDRN_REQUIRE(!pnp_conv || pi < 3, "run_stage: pnp_conv index out of range (0..2)");
  GDRN_REQUIRE(!down || (ds >= 1 && ds <= 3), "run_stage: down index out of range (1..3)");
  GDRN_REQUIRE(!block || (bs <= 3 && bi < a.depths[bs]), "run_stage: block index out of range for this arch");
  const bool backbone = stem || down || block;
  GDRN_REQUIRE(!(stem || out_conv || pnp_fc) || !raw_out, "run_stage: this stage has no conv output / operand");
  GDRN_REQUIRE(!(backbone || out_conv || pnp_fc) || !gn_stats_out, "run_stage: this stage has no GroupNorm sums");
  if (out_conv) {
    GDRN_REQUIRE(roi_extents && roi_coord_2d, "run_stage: out_conv needs roi_extents and roi_coord_2d");
    GDRN_REQUIRE(roi_classes || m->num_classes == 1, "run_stage: roi_classes is NULL but the head is class-aware");
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int B = batch, PR = m->precise;
  void* wbase = reinterpret_cast<void*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~(uintptr_t)1023);
  Workspace w = carve(m, B, wbase);
  m->prof_used = 0;
  m->prof_cat.clear();
  GDRN_CHECK_CUDA(cudaMemsetAsync(w.gn_stats, 0, w.zero_bytes, st));
  // fp32 -> the stage's operand format (bf16 or [hi | lo] split rows) and back
  auto encode = [&](__nv_bfloat16* dst, long long rows, int C) {
    return PR ? launch_cast_split(in, dst, rows, C, st) : launch_cast_bf16(in, dst, rows * C, st);
  };
  auto decode_to = [&](float* dst, const __nv_bfloat16* src, long long rows, int C) {
    return PR ? launch_split_to_f32(src, dst, rows, C, st) : launch_bf16_to_f32(src, dst, rows * C, st);
  };
  auto decode = [&](const __nv_bfloat16* src, long long rows, int C) { return decode_to(out, src, rows, C); };
  auto copy_f32 = [&](float* dst, const void* src, long long n) {
    GDRN_CHECK_CUDA(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st));
    return GDRN_OK;
  };
  const void* raw = nullptr;   // pre-GroupNorm conv output (fp32 in split-bf16 mode, bf16 otherwise) and its element count
  long long raw_n = 0;
  // backbone: the fp32 residual stream w.X is the stage's input and output in both modes; raw_out is the GEMM A operand
  // the LayerNorm kernel wrote (w.A)
  if (stem) {
    RC(stage_stem(m, w, B, in, st));
    RC(copy_f32(out, w.X, (long long)B * 64 * 64 * a.cp[0]));
  } else if (down) {
    const int r = 64 >> ds, Ci = a.cp[ds - 1];
    RC(copy_f32(w.X, in, (long long)B * 4 * r * r * Ci));
    RC(stage_downsample(m, w, B, ds, st));
    RC(copy_f32(out, w.X, (long long)B * r * r * a.cp[ds]));
    if (raw_out) RC(decode_to(raw_out, w.A, (long long)B * r * r, 4 * Ci));
  } else if (block) {
    const int r = 64 >> bs, C = a.cp[bs];
    RC(copy_f32(w.X, in, (long long)B * r * r * C));
    RC(stage_block(m, w, B, bs, bi, st));
    RC(copy_f32(out, w.X, (long long)B * r * r * C));
    if (raw_out) RC(decode_to(raw_out, w.A, (long long)B * r * r, C));
  } else if (deconv) {
    const int C3 = m->arch.cp[3];
    RC(encode(w.feat, (long long)B * 64, C3));
    RC(stage_deconv(m, w, B, w.feat, w.P, st));
    RC(decode(w.P, (long long)B * 256, 256));
    raw = w.R; raw_n = (long long)B * 256 * 256;
  } else if (head_conv) {
    const int h = 16 << (li / 2), ho = (li == 1 || li == 3) ? 2 * h : h;
    RC(encode(w.P, (long long)B * h * h, 256));
    RC(stage_head_conv(m, w, B, li, w.P, w.Q, st));
    RC(decode(w.Q, (long long)B * ho * ho, 256));
    raw = w.R; raw_n = (long long)B * h * h * 256;
  } else if (out_conv) {
    RC(encode(w.P, (long long)B * 4096, 256));
    RC(stage_out_conv(m, w, B, w.P, roi_classes, roi_extents, roi_coord_2d, maps, st));
    RC(decode(w.pnp_in, (long long)B * 4096, 128));
  } else if (pnp_conv) {
    const int ires = 64 >> pi, ores = ires / 2;
    __nv_bfloat16* src = pi == 0 ? w.pnp_in : w.pP;
    RC(encode(src, (long long)B * ires * ires, 128));
    RC(stage_pnp_conv(m, w, B, pi, src, st));
    if (PR && pi == 2) RC(copy_f32(out, w.pF, (long long)B * ores * ores * 128));
    else RC(decode(w.pP, (long long)B * ores * ores, 128));
    raw = w.pR; raw_n = (long long)B * ores * ores * 128;
  } else {
    if (PR) RC(copy_f32(w.pF, in, (long long)B * 8192));
    else RC(launch_cast_bf16(in, w.pP, (long long)B * 8192, st));
    RC(stage_pnp_fc(m, w, B, st));
    RC(copy_f32(out, w.fout, (long long)B * 16));
  }
  if (raw_out && raw) {
    if (PR) RC(copy_f32(raw_out, raw, raw_n));
    else RC(launch_bf16_to_f32(reinterpret_cast<const __nv_bfloat16*>(raw), raw_out, raw_n, st));
  }
  if (gn_stats_out) GDRN_CHECK_CUDA(cudaMemcpyAsync(gn_stats_out, w.gn_stats, w.zero_bytes, cudaMemcpyDeviceToDevice, st));
  return GDRN_OK;
}
