"""Per-shape timing of the split-bf16 GEMMs of the ConvNeXt stages (gdrn_gemm_x3): us / call and executed TFLOP/s (3 products).
Usage (on the GPU): python tools/x3_shapes_bench.py [--trace]"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gdrnpp_bop2022_b200 import _lib as L  # noqa: E402

SHAPES = [  # (name, M, N, K, block_n, epi)
    ("s0 fc1", 262144, 512, 128, 256, 1), ("s0 fc2", 262144, 128, 512, 128, 2),
    ("s1 fc1", 65536, 1024, 256, 256, 1), ("s1 fc2", 65536, 256, 1024, 256, 2),
    ("s2 fc1", 16384, 2048, 512, 256, 1), ("s2 fc2", 16384, 512, 2048, 256, 2),
    ("s3 fc1", 4096, 4096, 1024, 256, 1), ("s3 fc2", 4096, 1024, 4096, 256, 2),
    ("down1", 65536, 256, 512, 256, 0), ("down2", 16384, 512, 1024, 256, 0), ("down3", 4096, 1024, 2048, 256, 0),
]


def main():
    dev = torch.device("cuda:0")
    lib = L.lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = []
    for name, M, N, K, bn, epi in SHAPES:
        g = torch.Generator().manual_seed(M + N)
        A = torch.randn(M, 2 * K, generator=g).to(dev).bfloat16()
        W = (torch.randn(N, 2 * K, generator=g) / np.sqrt(K)).to(dev).bfloat16()
        bias, gamma = torch.randn(N).to(dev), torch.rand(N).to(dev)
        o = torch.zeros((M, 2 * N), dtype=torch.bfloat16, device=dev) if epi == 1 else torch.zeros((M, N), dtype=torch.float32, device=dev)
        if epi == 2:   # in-place residual entry (the fc2 GEMMs of the forward)
            flags = torch.zeros(8192, dtype=torch.int32, device=dev)
            call = lambda: L.check(lib.gdrn_gemm_x3_ksplit(L.ptr(A), L.ptr(W), L.ptr(bias), L.ptr(gamma), L.ptr(o), M, N, K, bn,
                                                           L.ptr(flags), 8192, L.current_stream()), "gemm_x3_ksplit")
        else:
            call = lambda: L.check(lib.gdrn_gemm_x3(L.ptr(A), L.ptr(W), L.ptr(bias), L.ptr(gamma), L.ptr(o), L.ptr(o), M, N, K, epi, bn,
                                                    L.current_stream()), "gemm_x3")
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        tot, n = 0.0, 10
        for _ in range(n):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); call(); e1.record(); e1.synchronize()
            tot += e0.elapsed_time(e1)
        us = tot / n * 1e3
        out.append({"shape": name, "M": M, "N": N, "K": K, "us": round(us, 1), "exec_tflops": round(3 * 2.0 * M * N * K / us / 1e6, 1)})
        print(out[-1], flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
