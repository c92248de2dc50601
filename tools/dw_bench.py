"""Depthwise 7x7 + LayerNorm kernels at the four ConvNeXt stage shapes (B = 64): us / launch of the one-tile-per-CTA
cluster kernel (variant 0) and the persistent ping-pong kernel (variant 1), bf16 and split output.
Usage (on the GPU): python tools/dw_bench.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gdrnpp_bop2022_b200 import _lib as L  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    lib = L.lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    B = 64
    for H, C in ((64, 128), (32, 256), (16, 512)):
        g = torch.Generator().manual_seed(C)
        x = torch.randn(B, H, H, C, generator=g).to(dev)
        w49c = (torch.randn(49, C, generator=g) / 7).to(dev)
        bias, lw, lb = torch.randn(C).to(dev) * 0.1, torch.rand(C).to(dev) + 0.5, torch.randn(C).to(dev) * 0.1
        for split in (0, 1):
            o = torch.empty((B * H * H, (2 if split else 1) * C), dtype=torch.bfloat16, device=dev)
            for variant in (0, 1):
                call = lambda: L.check(lib.gdrn_dwconv_ln(L.ptr(x), L.ptr(w49c), L.ptr(bias), L.ptr(lw), L.ptr(lb), L.ptr(o), B, H, H, C, 1e-6,
                                                          split, variant, L.current_stream()), "dwconv")
                for _ in range(3):
                    call()
                torch.cuda.synchronize()
                tot, n = 0.0, 10
                for _ in range(n):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); call(); e1.record(); e1.synchronize()
                    tot += e0.elapsed_time(e1)
                print("dw %dx%d C=%d split=%d variant=%d: %.1f us" % (H, H, C, split, variant, tot / n * 1e3), flush=True)


if __name__ == "__main__":
    main()
