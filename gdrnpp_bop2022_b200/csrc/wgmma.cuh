// wgmma.mma_async m64nNk16, bf16 x bf16 -> fp32, both operands K-major in shared memory (sm_90a).
// D (64 x N fp32, N / 2 registers per thread of the warpgroup) = (accumulate ? D : 0) + A (64 x 16) * B^T (N x 16).
// Accumulator fragment: register i of thread t (warp w = t / 32 of the warpgroup, lane l) holds
//   row w * 16 + l / 4 + 8 * ((i / 2) % 2), column (i / 4) * 8 + (l % 4) * 2 + i % 2.
#pragma once
#include <stdint.h>

#define GDRN_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                   "+f"(d[i + 6]), "+f"(d[i + 7])

namespace ptx {

template <int N>
struct Wgmma;

template <>
struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7"
        "}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
        : GDRN_F8(0)
        : "l"(a), "l"(b), "r"(accumulate)
        : "memory");
  }
};

template <>
struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : GDRN_F8(0), GDRN_F8(8), GDRN_F8(16), GDRN_F8(24)
        : "l"(a), "l"(b), "r"(accumulate)
        : "memory");
  }
};

template <>
struct Wgmma<80> {
  static __device__ __forceinline__ void mma(float (&d)[40], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39"
        "}, %40, %41, p, 1, 1, 0, 0;\n\t}\n"
        : GDRN_F8(0), GDRN_F8(8), GDRN_F8(16), GDRN_F8(24), GDRN_F8(32)
        : "l"(a), "l"(b), "r"(accumulate)
        : "memory");
  }
};

template <>
struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : GDRN_F8(0), GDRN_F8(8), GDRN_F8(16), GDRN_F8(24), GDRN_F8(32), GDRN_F8(40), GDRN_F8(48), GDRN_F8(56)
        : "l"(a), "l"(b), "r"(accumulate)
        : "memory");
  }
};

}  // namespace ptx

#undef GDRN_F8
