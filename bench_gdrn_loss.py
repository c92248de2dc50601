"""Time forward + backward of the GDRN training loss: gdrn_loss.gdrn_loss (csrc/gdrn_loss.cu) against the fp32 CUDA
restatement of the reference's gdrn_loss (oracle/gdrn_loss_oracle.py: the same torch ops and the same per-ROI host loop
that picks the closest symmetric GT rotation).

Shapes: B = 36 and 48 (the shipped IMS_PER_BATCH values), 64 regions on 64 x 64 maps, 3000 PM points (NUM_PM_POINTS),
every ROI with K = 0, 2 or 628 symmetry rotations (none; a discrete half turn with the identity; a continuous symmetry
with a flip at max_sym_disc_step = 0.01), PM_LOSS_SYM on.  Every shape is warmed up, the two arms alternate, each timed
over windows of at least --window seconds with a synchronised host clock; the losses of both arms are compared first.
Prints one JSON line with the card's name and power limit read in the same run.

  python bench_gdrn_loss.py [--window 1.0] [--quick]
"""
import argparse
import json
import subprocess
import time

import torch

from gdrnpp_bop2022_b200 import gdrn_loss as G
from oracle import gdrn_loss_oracle as O

ARGS = ("out_mask_vis", "out_mask_full", "gt_mask_trunc", "gt_mask_visib", "gt_mask_obj", "gt_mask_full", "out_x",
        "out_y", "out_z", "gt_xyz", "gt_xyz_bin", "out_region", "gt_region", "out_rot", "gt_rot", "out_trans",
        "gt_trans", "out_centroid", "out_trans_z", "gt_trans_ratio", "gt_points", "sym_infos", "extents")
SYMS = {0: "none", 2: "two", 628: "cont"}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def step(arm, cfg, d):
    for k in O.DENSE + O.SMALL:
        d[k].grad = None
    if arm == "ours":
        losses = G.gdrn_loss(None, cfg, **{k: d[k] for k in ARGS})
    else:
        losses = O.gdrn_loss(cfg, d)
    sum(losses.values()).backward()
    return losses


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--quick", action="store_true", help="one small shape (a rehearsal, not a measurement)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gdrn_loss.py needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = O.make_cfg()
    shapes = [(4, 2)] if args.quick else [(B, K) for B in (36, 48) for K in (0, 2, 628)]
    tables = O.sym_tables()
    rows = []
    for B, K in shapes:
        d = O.to(O.make_case(seed=B + K, B=B, syms=(SYMS[K],), N=3000, tables=tables), torch.float32, dev)
        ours = step("ours", cfg, d)
        ref = step("ref", cfg, d)
        agree = max(abs(float(ours[k].detach()) - float(ref[k].detach())) / max(abs(float(ref[k].detach())), 1e-12)
                    for k in ref)
        if agree > 1e-4:
            raise SystemExit(f"losses disagree at B={B} K={K}: relative {agree:.2e}")
        t = {"ours": [], "ref": []}
        for _ in range(3):   # alternate the arms
            for arm in ("ours", "ref"):
                t[arm].append(timed(lambda: step(arm, cfg, d), args.window))
        t_ours, t_ref = min(t["ours"]), min(t["ref"])
        rows.append({"B": B, "K": K, "ms": round(t_ours, 4), "baseline_ms": round(t_ref, 3),
                     "speedup": round(t_ref / t_ours, 1), "ms_all": [round(x, 4) for x in t["ours"]],
                     "baseline_ms_all": [round(x, 3) for x in t["ref"]], "max_rel_loss_diff": float(f"{agree:.2e}")})
        del d
        torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "gdrn_loss", "what": "gdrn_loss forward + backward, fp32, R = 64, 64x64 maps, N = 3000, "
                      "PM_LOSS_SYM on", "gpu": name, "power_limit": power, "window_s": args.window, "rows": rows}))


if __name__ == "__main__":
    main()
