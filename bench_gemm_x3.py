#!/usr/bin/env python
"""bench_gemm_x3.py -- the split-bf16 GEMM (gdrn_gemm_x3, parity mode) at the rank-2 shapes of the ConvNeXt stage-1..3 MLPs
of bench.py's B = 64 forward, with the tile widths the forward picks for them.

  python bench_gemm_x3.py [--reps R]    CUDA-event time per call (L2 flushed before each call: the forward reads A from
                                        HBM), algorithmic (2MNK) and executed (3 products) TFLOP/s, card name, power limit
                                        and the SM clock sampled while each shape runs

The conv GEMMs (head 3x3, deconv, Patch-PnP) have no stand-alone entry; bench.py's roofline.gemm_ms_per_step covers them.
Prints one JSON line at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SHAPES = [  # (name, M, N, K, epilogue): fc1 = GELU -> split bf16 hidden, fc2 = in-place layer-scale residual
    ("stage-1 fc1", 65536, 1024, 256, 1), ("stage-1 fc2", 65536, 256, 1024, 2),
    ("stage-2 fc1", 16384, 2048, 512, 1), ("stage-2 fc2", 16384, 512, 2048, 2),
    ("stage-3 fc1", 4096, 4096, 1024, 1), ("stage-3 fc2", 4096, 1024, 4096, 2),
]


def pick_bn(N, M, num_sms):
    """The forward's tile width (model.cu pick_bn): the widest one N divides into that still yields half a wave of CTAs."""
    m_tiles = (M + 127) // 128
    bn = 256 if N % 256 == 0 else (128 if N % 128 == 0 else 64)
    while bn > 64 and m_tiles * (N // bn) < num_sms // 2:
        bn >>= 1
    return bn


def card_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    parts = [p.strip() for p in q.stdout.strip().split(",")]
    if q.returncode != 0 or len(parts) < 3:
        return {"nvidia_smi": "unavailable"}
    return {"nvidia_smi_name": parts[0], "power_limit_w": float(parts[1]), "sm_max_mhz": float(parts[2])}


def make_operands(M, N, K, epi, dev):
    import numpy as np
    import torch

    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, 2 * K, generator=g).to(dev).bfloat16()
    W = (torch.randn(N, 2 * K, generator=g) / np.sqrt(K)).to(dev).bfloat16()
    bias, gamma = torch.randn(N, generator=g).to(dev), torch.rand(N, generator=g).to(dev)
    if epi == 1:
        out = torch.zeros((M, 2 * N), dtype=torch.bfloat16, device=dev)
    else:
        out = torch.zeros((M, N), dtype=torch.float32, device=dev)
    return A, W, bias, gamma, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30, help="timed calls per shape (median reported)")
    args = ap.parse_args()
    import torch

    from bench import ClockSampler
    from gdrnpp_bop2022_b200 import _lib as L

    assert torch.cuda.is_available(), "bench_gemm_x3.py needs a GPU"
    dev = torch.device("cuda:0")
    lib = L.lib()
    num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    info = {"card": torch.cuda.get_device_name(dev), **card_info()}
    print(json.dumps(info), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    records = []
    for name, M, N, K, epi in SHAPES:
        bn = pick_bn(N, M, num_sms)
        A, W, bias, gamma, out = make_operands(M, N, K, epi, dev)

        def call():
            L.check(lib.gdrn_gemm_x3(L.ptr(A), L.ptr(W), L.ptr(bias), L.ptr(gamma), L.ptr(out), L.ptr(out), M, N, K, epi, bn,
                                     L.current_stream()), "gemm_x3")

        # warm up for half a second: it settles the clock and lets nvidia-smi deliver its first samples
        sampler = ClockSampler(0)
        sampler.start()
        t_end = time.perf_counter() + 0.5
        while time.perf_counter() < t_end:
            for _ in range(10):
                call()
            torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        clocks = sampler.stop()
        times.sort()
        ms = times[len(times) // 2]
        tflops = 2.0 * M * N * K / (ms * 1e-3) / 1e12
        rec = {"shape": name, "M": M, "N": N, "K": K, "block_n": bn, "epi": epi, "us_median": round(ms * 1e3, 1),
               "us_min": round(times[0] * 1e3, 1), "us_max": round(times[-1] * 1e3, 1),
               "algorithmic_tflops": round(tflops, 1), "executed_tflops": round(3 * tflops, 1),
               "sm_mhz_median": clocks.get("sm_mhz"), "clock_event_reasons": clocks.get("reasons")}
        records.append(rec)
        print(json.dumps(rec), flush=True)
        del A, W, bias, gamma, out
    total_us = sum(r["us_median"] for r in records)
    print(json.dumps({"bench": "gemm_x3", **info, "total_us": round(total_us, 1), "shapes": records}))


if __name__ == "__main__":
    main()
