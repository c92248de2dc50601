"""Time the parameter update of both trainers: ranger.Ranger (csrc/train_step.cu) against the fp32 restatement of the
reference's Ranger.step (oracle/ranger_oracle.py: the same torch ops, eager on the GPU), on the full GDRN
(ConvNeXt-base + heads, 380 tensors) and YOLOX-X (456 tensors) parameter sets, for a plain step and a lookahead step;
and ema.ModelEMA.update against the reference's two torch ops per entry on the YOLOX-X state (748 floating entries).

Both arms start from the same state, past the RAdam warm-up (adaptive branch); a plain step uses k = 10**9, a lookahead
step k = 1.  Both arms' results are compared first.  Every shape is warmed up, the arms alternate, each is timed over
windows of at least --window seconds with a synchronised host clock.  Also reported per arm: the host enqueue time
(the call alone, after a synchronise), the device time of one step (CUDA events), and for ours the update kernel's own
time from torch.profiler in a separate pass, with the bytes it must move (computed from the shapes) and the achieved
rate against the H100 SXM data-sheet 3.35 TB/s.  Prints one JSON line with the card's name and power limit read in the
same run.

  python bench_ranger.py [--window 1.0] [--quick]
"""
import argparse
import copy
import json
import subprocess
import time

import torch

from gdrnpp_bop2022_b200.ema import ModelEMA
from gdrnpp_bop2022_b200.ranger import Ranger
from oracle import ranger_oracle as O

PEAK_BPS = 3.35e12
PLAIN_K = 10 ** 9


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def param_shapes(which, quick):
    if which == "gdrn":
        from gdrnpp_bop2022_b200.synthetic import state_dict_shapes

        shapes, kw = list(state_dict_shapes().values()), dict(lr=8e-4, weight_decay=0.01)
    else:
        from gdrnpp_bop2022_b200.yolox_model import YOLOX

        shapes, kw = [tuple(p.shape) for p in YOLOX(1.33, 1.25, 8).parameters()], dict(lr=0.001, weight_decay=0)
    if quick:
        shapes = [tuple(max(1, s // 16) for s in sh) for sh in shapes]
    return shapes, kw


def step_bytes(shapes, threshold, lookahead):
    """HBM bytes one fused step must move: read g, p, m, v; write p, m, v, and g when centralised; slow both ways on
    a lookahead step."""
    total = 0
    for sh in shapes:
        n = 1
        for s in sh:
            n *= s
        per = 16 + 12 + (4 if len(sh) > threshold else 0) + (8 if lookahead else 0)
        total += n * per
    return total


def timed(fn, window):
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= window:
            return dt / n * 1e3


def enqueue_and_device_ms(fn, reps=10):
    host, dev = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        fn()
        host.append((time.perf_counter() - t0) * 1e3)
        e1.record()
        torch.cuda.synchronize()
        dev.append(e0.elapsed_time(e1))
    return min(host), min(dev)


def kernel_ms(fn, names, reps=10):
    """Mean device time per call of the kernels whose names contain one of ``names``, from torch.profiler."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names))
    return us / reps / 1e3


def make_arm(cls, shapes, kw, grads, dev):
    gen = torch.Generator(device=dev).manual_seed(1)
    ps = [torch.nn.Parameter(0.02 * torch.randn(s, generator=gen, device=dev)) for s in shapes]
    opt = cls(ps, **kw)
    for i in range(7):   # past the warm-up: the adaptive branch from here on
        for p, g in zip(ps, grads[i % 2]):
            p.grad = g.clone()
        opt.step()
    return ps, opt


def bench_set(which, window, quick, dev):
    shapes, kw = param_shapes(which, quick)
    gen = torch.Generator(device=dev).manual_seed(2)
    grads = [[1e-3 * torch.randn(s, generator=gen, device=dev) for s in shapes] for _ in range(2)]
    arms = {"ours": make_arm(Ranger, shapes, kw, grads, dev), "ref": make_arm(O.RefRanger, shapes, kw, grads, dev)}
    threshold = arms["ours"][1].gc_gradient_threshold

    def set_k(opt, k):
        for g in opt.param_groups:
            g["k"] = k

    def step_fn(arm):
        ps, opt = arms[arm]

        def fn():   # the gradients stay in place: centralising a centralised gradient costs the same
            opt.step()
        return fn

    # agreement: one lookahead step from the same state, max error relative to the largest magnitude per tensor
    a, b = arms["ours"], arms["ref"]
    with torch.no_grad():
        for pa, pb in zip(a[0], b[0]):
            pa.copy_(pb)
            for k in O.STATE_KEYS:
                a[1].state[pa][k].copy_(b[1].state[pb][k])
    for _, opt in arms.values():
        set_k(opt, 1)
    for (ps, opt) in arms.values():
        for p, g in zip(ps, grads[0]):
            p.grad.copy_(g)
        opt.step()
    agree = max(((pa.detach() - pb.detach()).abs().max() / pb.detach().abs().max().clamp_min(1e-30)).item()
                for pa, pb in zip(a[0], b[0]))
    if agree > 1e-5:
        raise SystemExit(f"{which}: the arms disagree, relative {agree:.2e}")
    rows = []
    for mode, k in (("plain", PLAIN_K), ("lookahead", 1)):
        for _, opt in arms.values():
            set_k(opt, k)
        t = {"ours": [], "ref": []}
        for arm in ("ours", "ref"):   # warm-up
            step_fn(arm)()
        for _ in range(3):
            for arm in ("ours", "ref"):
                t[arm].append(timed(step_fn(arm), window))
        row = {"set": which, "tensors": len(shapes), "mode": mode, "ms": round(min(t["ours"]), 3),
               "baseline_ms": round(min(t["ref"]), 3), "speedup": round(min(t["ref"]) / min(t["ours"]), 1),
               "ms_all": [round(x, 3) for x in t["ours"]], "baseline_ms_all": [round(x, 3) for x in t["ref"]]}
        for arm in ("ours", "ref"):
            host, devt = enqueue_and_device_ms(step_fn(arm))
            row[("" if arm == "ours" else "baseline_") + "enqueue_ms"] = round(host, 3)
            row[("" if arm == "ours" else "baseline_") + "device_ms"] = round(devt, 3)
        kms = kernel_ms(step_fn("ours"), ("rs_step_kernel", "rs_long_means_kernel"))
        nbytes = step_bytes(shapes, threshold, mode == "lookahead")
        row.update({"kernel_ms": round(kms, 4), "bytes_per_step": nbytes,
                    "kernel_GBps": round(nbytes / (kms * 1e-3) / 1e9, 1),
                    "share_of_3.35TBps": round(nbytes / (kms * 1e-3) / PEAK_BPS, 3)})
        rows.append(row)
    row0 = rows[0]
    row0["max_rel_diff"] = float(f"{agree:.2e}")
    del arms, grads
    torch.cuda.empty_cache()
    return rows


def bench_ema(window, quick, dev):
    from gdrnpp_bop2022_b200.yolox_model import YOLOX

    torch.manual_seed(0)
    model = YOLOX(0.33, 0.25, 8) if quick else YOLOX(1.33, 1.25, 8)
    model = model.to(dev)
    ours = ModelEMA(model, 0.9998, updates=3000)
    ref_ema = copy.deepcopy(ours.ema)
    ref_sd = ref_ema.state_dict()
    counter = {"n": 3000}

    def ref_fn():   # the reference's update: both state dicts, then two ops per floating entry
        counter["n"] += 1
        O.ema_update(ref_ema.state_dict(), model.state_dict(), O.ema_decay(0.9998, counter["n"]))

    O.perturb_model(model, 0, 1)
    ours.update(model)
    ref_fn()
    for k, v in ours.ema.state_dict().items():
        if not torch.equal(v, ref_sd[k]):
            raise SystemExit(f"EMA differs from the reference ops at {k}")
    fns = {"ours": lambda: ours.update(model), "ref": ref_fn}
    t = {"ours": [], "ref": []}
    for _ in range(3):
        for arm in ("ours", "ref"):
            t[arm].append(timed(fns[arm], window))
    n_float = sum(v.numel() for v in ref_sd.values() if v.is_floating_point())
    nbytes = 12 * n_float
    row = {"set": "yolox_ema", "entries": sum(1 for v in ref_sd.values() if v.is_floating_point()), "ms":
           round(min(t["ours"]), 3), "baseline_ms": round(min(t["ref"]), 3),
           "speedup": round(min(t["ref"]) / min(t["ours"]), 1), "bit_exact": True}
    for arm in ("ours", "ref"):
        host, devt = enqueue_and_device_ms(fns[arm])
        row[("" if arm == "ours" else "baseline_") + "enqueue_ms"] = round(host, 3)
        row[("" if arm == "ours" else "baseline_") + "device_ms"] = round(devt, 3)
    kms = kernel_ms(fns["ours"], ("ema_kernel",))
    row.update({"kernel_ms": round(kms, 4), "bytes_per_step": nbytes,
                "kernel_GBps": round(nbytes / (kms * 1e-3) / 1e9, 1),
                "share_of_3.35TBps": round(nbytes / (kms * 1e-3) / PEAK_BPS, 3)})
    return [row]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--quick", action="store_true", help="shapes / 16 (a rehearsal, not a measurement)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ranger.py needs a CUDA device")
    dev = torch.device("cuda:0")
    rows = bench_set("gdrn", args.window, args.quick, dev) + bench_set("yolox", args.window, args.quick, dev)
    rows += bench_ema(args.window, args.quick, dev)
    name, power = card()
    print(json.dumps({"bench": "ranger", "what": "Ranger.step (fp32, GC on, adaptive branch) and ModelEMA.update",
                      "gpu": name, "power_limit": power, "window_s": args.window, "rows": rows}))


if __name__ == "__main__":
    main()
