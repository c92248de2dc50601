"""YOLOX-X (depth 1.33, width 1.25, 8 classes, 640 x 640) forward: images/s and per-call latency of YOLOX.forward on the
CUDA kernels (B = 1 replayed as a captured CUDA graph, B = 8 and 32 eager) in both precisions, next to the same network
in torch eager with cuDNN (the fp64 oracle's functional forward run in fp32 with TF32 off, and in fp16 like the
reference's half_test=True).  Weights are synthetic (gdrnpp_bop2022_b200.synthetic.make_yolox_state_dict).

The arithmetic floor is 281 GFLOP per image (140.5 GMAC) over the data sheet's 989 TFLOP/s dense bf16 (H100 SXM):
0.28 ms per image in bf16 and three times that in bf16x3 (three bf16 products per MAC).  It is a data-sheet floor, not
a measured rate.  Prints one JSON line per configuration, with the card name and power limit.

  python bench_yolox.py [--min-window-ms 1000] [--batches 1,8,32]

Each number is the median of three timed windows of at least --min-window-ms each, with the min and max beside it.
"""
import argparse
import json
import subprocess

import torch

GFLOP_PER_IMAGE = 281.0
PEAK_TFLOPS_BF16 = 989.0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:   # noqa: BLE001 -- the name is informative only
        q = torch.cuda.get_device_name()
    return q


def timed(fn, iters, warmup=3, repeats=3):
    """-> (median, min, max) ms per call over ``repeats`` windows of ``iters`` calls (CUDA events)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b) / iters)
    per.sort()
    return per[len(per) // 2], per[0], per[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-ms", type=float, default=1000.0, help="each timed window lasts at least this long")
    ap.add_argument("--batches", default="1,8,32")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_yolox.py needs a GPU"
    from gdrnpp_bop2022_b200.synthetic import make_yolox_state_dict
    from gdrnpp_bop2022_b200.yolox_model import YOLOX
    from oracle.yolox_oracle import yolox_forward

    name = card()
    dev = torch.device("cuda")
    sd = make_yolox_state_dict(yolox_forward, 1.33, 1.25, 8, seed=0, device="cuda")
    batches = [int(b) for b in args.batches.split(",")]
    rows = []

    def run(fn):
        fn()
        torch.cuda.synchronize()
        t = timed(fn, 3, warmup=1, repeats=1)[0]   # rough per-call time: size the windows to min_window_ms
        return timed(fn, max(5, int(args.min_window_ms / max(t, 1e-3)) + 1))

    def report(impl, precision, B, stats):
        ms, lo, hi = stats
        floor = GFLOP_PER_IMAGE * B / PEAK_TFLOPS_BF16 * (3 if precision == "bf16x3" else 1)   # ms
        r = {"impl": impl, "precision": precision, "batch": B, "ms_per_call": round(ms, 3),
             "ms_min_max": [round(lo, 3), round(hi, 3)],
             "images_per_s": round(1000.0 * B / ms, 1),
             "share_of_bf16_floor": round(floor / ms, 3) if precision in ("bf16", "bf16x3") else None, "card": name}
        rows.append(r)
        print(json.dumps(r), flush=True)

    for precision in ("bf16x3", "bf16"):
        m = YOLOX(1.33, 1.25, 8, max_batch=max(batches), precision=precision).eval()
        m.load_state_dict(sd)
        m.to(dev)
        for B in batches:
            x = torch.rand((B, 3, 640, 640), device=dev) * 255
            if B == 1:
                replay, _ = m.capture_graph(x)
                ms = run(replay)
            else:
                ms = run(lambda: m(x))
            report("cuda_kernels" + (" (graph)" if B == 1 else ""), precision, B, ms)
        del m
        torch.cuda.empty_cache()

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    for dtype, label in ((torch.float32, "fp32"), (torch.float16, "fp16")):
        sdt = {k: (v.to(dev, dtype) if v.is_floating_point() else v) for k, v in sd.items()}
        for B in batches:
            x = (torch.rand((B, 3, 640, 640), device=dev) * 255).to(dtype)
            with torch.no_grad():
                ms = run(lambda: yolox_forward(sdt, x, 1.33, 8))
            report("torch_eager_cudnn", label, B, ms)
    print(json.dumps({"summary": rows, "card": name}))


if __name__ == "__main__":
    main()
