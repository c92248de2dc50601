// DeepIM depth-reprojection optical flow.  Replaces core/csrc/flow/src/flow_cuda_kernel.cu:26-65
// (float instantiation; launch surface src/flow_cuda.cpp:30-42).
//
// HBM-bound elementwise op: 4 B depth read + 4 B gathered target depth + 12 B written per pixel = 20 B/pixel.
// Arithmetic is spelled out with explicit intrinsics in the contraction ptxas 12.9 / sm_90a applies to
// the reference source (a*K0 + b*K1 + c  ->  fma(a,K0, b*K1) + c), double-literal comparisons included,
// so flow/valid are bit-identical to the reference build.
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256)
flow_kernel(const float* __restrict__ depth_src, const float* __restrict__ depth_tgt, const float* __restrict__ KT,
            const float* __restrict__ Kinv, float* __restrict__ flow, float* __restrict__ valid, int batch, int height,
            int width) {
  const long long hw = (long long)height * width;
  const long long total = hw * batch;
  for (long long index = (long long)blockIdx.x * blockDim.x + threadIdx.x; index < total;
       index += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(index / hw);
    const unsigned rem = (unsigned)(index - (long long)b * hw);  // < H*W: 32-bit division below
    const int h = (int)(rem / (unsigned)width);
    const int w = (int)(rem - (unsigned)h * (unsigned)width);
    const float d = depth_src[index];
    float f0 = 0.f, f1 = 0.f, ok = 0.f;
    if ((double)d > 1E-3) {
      const float* ki = Kinv + b * 9;
      const float* kt = KT + b * 12;
      const float wf = (float)w, hf = (float)h;
      float x = __fmul_rn(__fadd_rn(__fmaf_rn(wf, ki[0], __fmul_rn(hf, ki[1])), ki[2]), d);
      float y = __fmul_rn(__fadd_rn(__fmaf_rn(wf, ki[3], __fmul_rn(hf, ki[4])), ki[5]), d);
      float xp = __fadd_rn(__fmaf_rn(d, kt[2], __fmaf_rn(x, kt[0], __fmul_rn(y, kt[1]))), kt[3]);
      float yp = __fadd_rn(__fmaf_rn(d, kt[6], __fmaf_rn(x, kt[4], __fmul_rn(y, kt[5]))), kt[7]);
      float zs = __fadd_rn(__fmaf_rn(d, kt[10], __fmaf_rn(x, kt[8], __fmul_rn(y, kt[9]))), kt[11]);
      float zp = (float)((double)zs + 1E-15);
      float wp = __fdiv_rn(xp, zp);
      float hp = __fdiv_rn(yp, zp);
      if (wp >= 0.f && wp <= (float)(width - 1) && hp >= 0.f && hp <= (float)(height - 1)) {
        int wi = (int)roundf(wp);
        int hi = (int)roundf(hp);
        float dt = depth_tgt[((long long)b * height + hi) * width + wi];
        if ((double)fabsf(__fsub_rn(zp, dt)) < 3E-3) {
          f0 = __fsub_rn(hp, hf);
          f1 = __fsub_rn(wp, wf);
          ok = 1.f;
        }
      }
    }
    flow[((long long)b * 2 + 0) * hw + (long long)h * width + w] = f0;
    flow[((long long)b * 2 + 1) * hw + (long long)h * width + w] = f1;
    valid[index] = ok;
  }
}

}  // namespace

extern "C" int flow_forward_cuda(const float* depth_src, const float* depth_tgt, const float* KT, const float* Kinv,
                                 float* flow, float* valid, int batch, int height, int width, void* stream) {
  GDRN_REQUIRE(batch > 0 && height > 0 && width > 0, "flow: empty input");
  long long total = (long long)batch * height * width;
  long long blocks = (total + 255) / 256;
  long long cap = (long long)gdrn_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  flow_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(depth_src, depth_tgt, KT, Kinv, flow, valid, batch, height,
                                                           width);
  GDRN_CHECK_CUDA(cudaGetLastError());
  gdrn_count_launch(1);
  return GDRN_OK;
}
