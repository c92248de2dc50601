"""Time the batched errors of eval_pose_results_more.py (bop_eval.rt_errors / proj_errors / ad) against the reference's
per-pair numpy functions, restated on the host (tests/test_pose_eval_more.py, pinned to the reference by
tests/golden/ref_pose_error_more.npz).

Workload: bench_bop_eval.py's synthetic YCB-V-like set (21 objects of 2,000-3,000 points, 8 of them symmetric and 5 of
those continuous, i.e. 314 symmetry transforms each), IMAGES images with 5 pairs each.  Timed error types:
  * reteS   rt_errors with the symmetry sets (the same call serves reS and teS)
  * projS   proj_errors with the symmetry sets: every point under every symmetry, the costly one
  * proj    proj_errors against the GT pose alone
  * AUCad   ad with no gate (ADI for the symmetric objects), the ABS* / AUC* path
The host numbers time the per-pair functions on a random subset of pairs and are scaled to the full set.

  python bench_pose_eval_more.py [--images 100] [--host-pairs 20] [--reps 5]
Prints one JSON line per error type with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_bop_eval import make_set, timed  # noqa: E402
from bench_per_object import card_info  # noqa: E402
from gdrnpp_bop2022_b200 import bop_eval  # noqa: E402
import test_bop_eval as B  # noqa: E402
import test_pose_eval_more as R  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--host-pairs", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pose_eval_more.py measures on a GPU"
    dev = torch.device("cuda:0")
    rs = np.random.RandomState(0)
    infos, points, pairs = make_set(rs, a.images)
    P = len(pairs)
    K = np.array([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]])
    models = bop_eval.PoseErrorModels(points, infos, device=dev)
    obj = [p[1] for p in pairs]
    Re, te, Rg, tg = (np.stack([p[k] for p in pairs]) for k in (2, 3, 4, 5))
    use_adi = np.array([bop_eval.is_symmetric("ycbv", o, infos[o]) for o in obj])
    card = card_info(0)
    gpu = {
        "reteS": timed(lambda: bop_eval.rt_errors(models, obj, Re, te, Rg, tg, True), a.reps),
        "projS": timed(lambda: bop_eval.proj_errors(models, obj, Re, te, Rg, tg, K, True), a.reps),
        "proj": timed(lambda: bop_eval.proj_errors(models, obj, Re, te, Rg, tg, K, False), a.reps),
        "AUCad": timed(lambda: bop_eval.ad(models, obj, Re, te, Rg, tg, use_adi) / 10, a.reps),
    }
    sub = rs.choice(P, min(a.host_pairs, P), replace=False)
    syms = {o: B.sym_stack(infos[o]) for o in infos}

    def host_time(f):
        t0 = time.perf_counter()
        for i in sub:
            f(i)
        return (time.perf_counter() - t0) / len(sub) * P

    host = {
        "reteS": host_time(lambda i: (R.re_sym_np(Re[i], Rg[i], syms[obj[i]]),
                                      R.te_sym_np(te[i], tg[i], Rg[i], syms[obj[i]]) / 10)),
        "projS": host_time(lambda i: R.arp_2d_sym_np(Re[i], te[i], Rg[i], tg[i], points[obj[i]], K, syms[obj[i]])),
        "proj": host_time(lambda i: R.arp_2d_np(Re[i], te[i], Rg[i], tg[i], points[obj[i]], K)),
        "AUCad": host_time(lambda i: (B.adi_np if use_adi[i] else B.add_np)(Re[i], te[i], Rg[i], tg[i], points[obj[i]]) / 10),
    }
    for k in gpu:
        print(json.dumps({"bench": "pose_eval_more", "error": k, "pairs": P, "images": a.images,
                          "gpu_ms": round(gpu[k] * 1e3, 3), "host_numpy_ms": round(host[k] * 1e3, 1),
                          "host_pairs_timed": len(sub), "card": card}))


if __name__ == "__main__":
    main()
