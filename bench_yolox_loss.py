"""Time forward + backward of the YOLOX training loss: yolox_loss.get_losses (csrc/yolox_loss.cu) against the fp32 CUDA
restatement of the reference's per-image loop (oracle/yolox_loss_oracle.py), with and without the reference's
per-image torch.cuda.empty_cache().

Shapes: T-LESS (C = 30), B = 8 and 64 (one GPU's share and the shipped total batch), square inputs of 448, 640 and 832
px (the ends and middle of the shipped random_size), 8, 30 and 120 GTs per image, use_l1 on.  Every shape is warmed up
and timed over windows of at least --window seconds with a synchronised host clock; the losses of both sides are
compared before timing.  Prints one JSON line with the card's name and power limit read in the same run.

  python bench_yolox_loss.py [--window 1.0] [--quick]
"""
import argparse
import json
import subprocess
import time

import torch

from gdrnpp_bop2022_b200 import yolox_loss as Y
from oracle import yolox_loss_oracle as O

C = 30


class Head:
    def __init__(self):
        self.num_classes, self.use_l1 = C, True
        self.iou_loss = type("IOUloss", (), {"loss_type": "iou"})()
        self.cls_loss_type = self.obj_loss_type = "bce"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def make(B, side, G, dev):
    xs, ys, es, labels, raw = O.make_case(100 + side + G + B, B, side, C, (G,) * B)
    mv = lambda ts: [t.to(dev) for t in ts]  # noqa: E731
    xs, ys, es = mv(xs), mv(ys), mv(es)
    outputs = O.decode(raw.to(dev), xs, ys, es)
    return xs, ys, es, labels.to(dev), outputs, raw[..., :4].to(dev)


def step(fn, head, xs, ys, es, labels, outputs, origin, **kw):
    out = outputs.detach().requires_grad_(True)
    org = origin.detach().requires_grad_(True)
    _, L = fn(head, None, xs, ys, es, labels, out, list(torch.split(org, [x.shape[1] for x in xs], 1)), out.dtype, **kw)
    (L["loss_iou"] + L["loss_conf"] + L["loss_cls"] + L["loss_l1"]).backward()
    return L


def timed(fn, window):
    fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= window:
            return dt / n * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--quick", action="store_true", help="one small shape (a rehearsal, not a measurement)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_yolox_loss.py needs a CUDA device")
    dev = torch.device("cuda:0")
    head = Head()
    shapes = [(8, 448, 8)] if args.quick else [(B, s, G) for B in (8, 64) for s in (448, 640, 832) for G in (8, 30, 120)]
    rows = []
    for B, side, G in shapes:
        data = make(B, side, G, dev)
        ours = step(Y.get_losses, head, *data)
        ref = step(O.get_losses, head, *data)
        agree = max(abs(float(ours[k].detach()) - float(ref[k].detach())) / max(abs(float(ref[k].detach())), 1e-12)
                    for k in ("loss_iou", "loss_conf", "loss_cls", "loss_l1"))
        if agree > 1e-3:
            raise SystemExit(f"losses disagree at B={B} side={side} G={G}: relative {agree:.2e}")
        t_ours = timed(lambda: step(Y.get_losses, head, *data), args.window)
        t_ref = timed(lambda: step(O.get_losses, head, *data), args.window)
        t_ref_ec = timed(lambda: step(O.get_losses, head, *data, empty_cache=True), args.window)
        rows.append({"B": B, "side": side, "gts": G, "anchors": int(data[4].shape[1]), "ms": round(t_ours, 4),
                     "baseline_ms": round(t_ref, 3), "baseline_empty_cache_ms": round(t_ref_ec, 3),
                     "speedup": round(t_ref / t_ours, 1), "speedup_empty_cache": round(t_ref_ec / t_ours, 1),
                     "max_rel_loss_diff": float(f"{agree:.2e}")})
        del data
        torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "yolox_loss", "what": "get_losses forward + backward, fp32, use_l1 on, C = 30",
                      "gpu": name, "power_limit": power, "window_s": args.window, "rows": rows}))


if __name__ == "__main__":
    main()
