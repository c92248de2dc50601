#!/usr/bin/env python
"""bench_per_object.py -- the per-object deployment on one H100: 21 class-agnostic convnext_base models (one per YCB-V
object, like the reference's configs/gdrn/ycbvSO/**) behind one PerObjectGDRN call.

  python bench_per_object.py [--steps 20] [--warmup 5] [--precision bf16x3|bf16]

Prints one JSON line: 5-ROI frame latency (5 different members per frame, CUDA graphs on), ROIs/s of 64-ROI batches
whose labels are spread over the 21 members (graphs on and eager), peak device memory, and the class-aware single
model on the same 64-ROI batches in the same run, with the card's name and power limit.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

BATCH = 64


def card_info(index):
    """Name and power limit of the card the numbers are measured on (read in the same run as the measurement)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=10)
        name, limit = [p.strip() for p in r.stdout.strip().split(",")[:2]]
        info.update(name=name, power_limit_w=float(limit))
    except Exception:  # noqa: BLE001
        pass
    return info


PER_OBJECT_MEMBERS = 21   # YCB-V: one network per object, like configs/gdrn/ycbvSO/**


def per_object_record(dev, precision, steps, warmup):
    """21 convnext_base class-agnostic members behind PerObjectGDRN (the reference's per-object deployment):
    (a) per-frame latency of 5-ROI frames whose ROIs belong to 5 different members, graphs on; (b) ROIs/s of
    64-ROI batches with labels drawn uniformly over the 21 members, graphs on (and eager); (c) peak device memory;
    (d) the class-aware single model on the same 64-ROI batches, same run.  Every member carries the same seeded weights
    (the work, and so the time, does not depend on their values); each has its own engine and weight buffers."""
    import numpy as np

    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg
    from gdrnpp_bop2022_b200.per_object import PerObjectGDRN
    from gdrnpp_bop2022_b200.synthetic import make_batch, make_state_dict

    K = PER_OBJECT_MEMBERS
    keys = ("roi_img", "roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "resize_ratios", "roi_extents")
    cfg = default_cfg()
    g = cfg.MODEL.POSE_NET.GEO_HEAD
    g.XYZ_CLASS_AWARE = g.MASK_CLASS_AWARE = g.REGION_CLASS_AWARE = False
    sd = make_state_dict(num_classes=1, seed=7)
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info(dev)
    reserved0 = torch.cuda.memory_reserved(dev)
    members = {}
    for label in range(K):   # parameters stay on the host: the engine holds the device copy of the weights
        members[label] = GDRN_DoubleMask(cfg, max_batch=BATCH, precision=precision)
        members[label].load_state_dict(sd)
    eager, graphed = PerObjectGDRN(members), PerObjectGDRN(members, use_cuda_graph=True)
    rs = np.random.RandomState(0)

    def fwd(pm, b, labels):
        return pm(b["roi_img"], roi_classes=labels, **{k: b[k] for k in keys if k != "roi_img"})

    # (b) 64-ROI batches over the 21 members (labels on the host, as the predictor's detections are)
    NB = 4
    big = [{k: v.to(dev) for k, v in make_batch(B=BATCH, seed=200 + i).items()} for i in range(NB)]
    big_labels = [torch.from_numpy(rs.randint(0, K, BATCH)) for _ in range(NB)]
    for i in range(NB):
        fwd(eager, big[i], big_labels[i])   # loads the 21 engines
    torch.cuda.synchronize()
    # device memory taken outside the torch allocator since the start: the 21 engines' weights (and stream objects)
    weights_bytes = free0 - torch.cuda.mem_get_info(dev)[0] - (torch.cuda.memory_reserved(dev) - reserved0)
    torch.cuda.reset_peak_memory_stats(dev)
    base_alloc = torch.cuda.memory_allocated(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(pm, n):
        e0.record()
        for i in range(n):
            fwd(pm, big[i % NB], big_labels[i % NB])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    n = max(steps // 2, 4)
    ms_b_eager = timed(eager, n)
    peak_eager = torch.cuda.max_memory_allocated(dev) - base_alloc
    for i in range(NB):
        fwd(graphed, big[i], big_labels[i])   # captures every (member, sub-batch size) of the four batches
    torch.cuda.synchronize()
    ms_b_graph = timed(graphed, n)
    # (a) 5-ROI frames, 5 different members each, graphs on: first capture (member, 1) for all 21 members
    frames = [{k: v.to(dev) for k, v in make_batch(B=5, seed=300 + i).items()} for i in range(8)]
    for f in range(5):
        fwd(graphed, frames[f], torch.tensor([(5 * f + j) % K for j in range(5)]))
    frame_labels = [torch.from_numpy(rs.choice(K, 5, replace=False)) for _ in range(64)]
    for i in range(warmup):
        fwd(graphed, frames[i % 8], frame_labels[i])
    torch.cuda.synchronize()
    lat = []
    for i in range(max(steps, 20)):
        t0 = time.perf_counter()
        fwd(graphed, frames[i % 8], frame_labels[i % 64])
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    lat.sort()
    torch.cuda.synchronize()
    used_bytes = total - torch.cuda.mem_get_info(dev)[0]
    n_graphs = len(graphed._graphs)
    graphed.release_graphs()
    del eager, graphed, members
    torch.cuda.empty_cache()
    # (d) the class-aware single model on the same 64-ROI batches
    single = GDRN_DoubleMask(default_cfg(), max_batch=BATCH, precision=precision)
    single.load_state_dict(make_state_dict())
    single.to(dev)
    caps = []
    for i in range(NB):
        b = dict(big[i], roi_classes=big_labels[i].to(dev))
        caps.append(single.capture_graph(b))
    e0.record()
    for i in range(n):
        caps[i % NB][0]()
    e1.record()
    torch.cuda.synchronize()
    ms_single = e0.elapsed_time(e1) / n
    del single, caps
    torch.cuda.empty_cache()
    return {
        "members": K, "arch": "convnext_base", "precision": precision, "card": card_info(dev.index),
        "frame5_ms": {"median": lat[len(lat) // 2], "p90": lat[int(len(lat) * 0.9)], "frames": len(lat),
                      "graph_replay": True,
                      "note": "5 ROIs of 5 different members per frame, host clock around forward + device synchronise"},
        "batch64": {"value": BATCH / ms_b_graph * 1e3, "unit": "ROIs/s", "ms_per_batch": ms_b_graph, "steps": n,
                    "graph_replay": True, "eager_value": BATCH / ms_b_eager * 1e3, "eager_ms_per_batch": ms_b_eager,
                    "labels": "uniform over the 21 members (4 fixed batches)"},
        "memory": {"torch_peak_bytes_eager_b64": peak_eager,
                   "engine_weight_bytes_approx": weights_bytes,
                   "device_used_bytes_at_end": used_bytes, "graphs_captured": n_graphs,
                   "note": "torch_peak: workspaces + gathered inputs + outputs of one eager 64-ROI call; device_used "
                           "includes the 21 engines, every captured graph's workspace and the rest of this process"},
        "class_aware_single_model": {"value": BATCH / ms_single * 1e3, "unit": "ROIs/s", "ms_per_batch": ms_single,
                                     "graph_replay": True, "note": "one 21-class model, the same 64-ROI batches"},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precision", default="bf16x3", choices=["bf16x3", "bf16"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_per_object.py needs a CUDA device (no CPU fallback for the product path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rec = per_object_record(dev, args.precision, args.steps, max(args.warmup, 3))
    print(json.dumps(dict({"record": "per_object"}, **rec)), flush=True)


if __name__ == "__main__":
    main()
