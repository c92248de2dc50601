"""Time the batched BOP pose errors (gdrnpp_bop2022_b200/bop_eval.py) against the reference's per-pair numpy loops,
restated on the host (tests/test_bop_eval.py, pinned to the reference by tests/golden/ref_pose_error.npz).

Workload: a synthetic YCB-V-like test split, 640x480, 21 objects (models_eval-sized point sets of 2,000-3,000 points,
the BOP symmetries of YCB-V's symmetric objects: 8 with discrete or continuous ones), IMAGES images with ~5 targets each
and one estimate per target (n_top = -1), so one pair per target.  VSD runs on stored depth maps (synthetic object
surfaces and scenes): this measures the per-pixel reduction, not rendering.  The host numbers time the same errors with
the reference's per-pair functions on a subset and are scaled to the full set.

  python bench_bop_eval.py [--images 100] [--host-pairs 20] [--reps 5]
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

from bench_per_object import card_info  # noqa: E402
from gdrnpp_bop2022_b200 import bop_eval  # noqa: E402
import test_bop_eval as R  # noqa: E402

H, W = 480, 640
N_OBJ = 21


def make_set(rs, images):
    infos, points = {}, {}
    for o in range(1, N_OBJ + 1):
        info = {"diameter": float(rs.uniform(80, 250))}
        if o in (13, 16, 19, 20, 21):   # continuous symmetry about z
            info["symmetries_continuous"] = [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]
        elif o in (1, 14, 18):
            info["symmetries_discrete"] = [[-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]]
        infos[o] = info
        points[o] = (rs.rand(rs.randint(2000, 3000), 3) - 0.5) * info["diameter"] * 0.6
    pairs = []
    for im in range(images):
        for o in rs.choice(np.arange(1, N_OBJ + 1), 5, replace=False):
            R_g = R._rand_rot(rs)
            t_g = np.array([rs.uniform(-150, 150), rs.uniform(-100, 100), rs.uniform(600, 1300)])
            dR = np.linalg.qr(np.eye(3) + rs.randn(3, 3) * 0.05)[0]
            dR *= np.sign(np.linalg.det(dR))
            pairs.append((im, int(o), dR @ R_g, t_g + rs.randn(3) * 10, R_g, t_g))
    return infos, points, pairs


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--host-pairs", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_bop_eval.py measures on a GPU"
    dev = torch.device("cuda:0")
    rs = np.random.RandomState(0)
    infos, points, pairs = make_set(rs, a.images)
    P = len(pairs)
    K = np.array([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]])
    models = bop_eval.PoseErrorModels(points, infos, device=dev)
    obj = [p[1] for p in pairs]
    Re, te, Rg, tg = (np.stack([p[k] for p in pairs]) for k in (2, 3, 4, 5))
    gate = np.array([bop_eval.spheres_overlap(te[i], tg[i], infos[obj[i]]["diameter"]) for i in range(P)])
    use_adi = np.array([bop_eval.is_symmetric("ycbv", o, infos[o]) for o in obj])
    # depth maps: one estimate / GT surface per pair, one scene per image
    ests, gts = np.zeros((P, H, W), np.float32), np.zeros((P, H, W), np.float32)
    for i, (im, o, _, t_e, _, t_g) in enumerate(pairs):
        r = infos[o]["diameter"] * 0.5 * K[0, 0] / t_g[2]
        c = (K[0, 0] * t_g[0] / t_g[2] + K[0, 2], K[1, 1] * t_g[1] / t_g[2] + K[1, 2])
        gts[i] = R._surface(rs, H, W, c[0], c[1], r, t_g[2], 0.3, -0.2)
        ests[i] = R._surface(rs, H, W, c[0] + 4, c[1] - 3, r, t_e[2], 0.25, -0.2)
    tests = np.full((a.images, H, W), 1800, np.float32)
    for i, (im, *_r) in enumerate(pairs):
        tests[im] = np.where((gts[i] > 0) & (gts[i] < tests[im]), gts[i], tests[im])
    tests[rs.rand(*tests.shape) < 0.05] = 0
    pair_img = np.array([p[0] for p in pairs], np.int32)
    vsd_gate = np.array([bop_eval.sphere_projections_overlap(infos[obj[i]]["diameter"] / 2, te[i], tg[i]) for i in range(P)])
    diam = np.array([infos[o]["diameter"] for o in obj])
    taus = R.BOP19_TAUS
    gd = {k: torch.from_numpy(v).to(dev) for k, v in (("e", ests), ("g", gts), ("t", tests))}
    idx = torch.arange(P, dtype=torch.int32, device=dev)
    pim, Kt, dt_, vg = (torch.from_numpy(x).to(dev) for x in (pair_img, np.stack([K] * P), diam, vsd_gate))
    card = card_info(0)
    gpu = {
        "vsd": timed(lambda: bop_eval.vsd(gd["e"], gd["g"], gd["t"], idx, idx, pim, Kt, dt_, taus, 15, True, vg), a.reps),
        "mssd+mspd": timed(lambda: bop_eval.mssd_mspd(models, obj, Re, te, Rg, tg, K, gate), a.reps),
        "ad": timed(lambda: bop_eval.ad(models, obj, Re, te, Rg, tg, use_adi, gate), a.reps),
    }
    sub = rs.choice(P, min(a.host_pairs, P), replace=False)
    syms = {o: R.sym_stack(infos[o]) for o in infos}

    def host_time(f):
        t0 = time.perf_counter()
        for i in sub:
            f(i)
        return (time.perf_counter() - t0) / len(sub) * P

    host = {
        "vsd": host_time(lambda i: R.vsd_np(ests[i], gts[i], tests[pair_img[i]], K, 15, taus, True, diam[i]) if vsd_gate[i] else None),
        "mssd+mspd": host_time(lambda i: (R.mssd_np(Re[i], te[i], Rg[i], tg[i], points[obj[i]], syms[obj[i]]) if gate[i] else None,
                                          R.mspd_np(Re[i], te[i], Rg[i], tg[i], K, points[obj[i]], syms[obj[i]]))),
        "ad": host_time(lambda i: ((R.adi_np if use_adi[i] else R.add_np)(Re[i], te[i], Rg[i], tg[i], points[obj[i]])
                                   if gate[i] else None)),
    }
    for k in gpu:
        print(json.dumps({"bench": "bop_eval", "error": k, "pairs": P, "images": a.images, "gpu_ms": round(gpu[k] * 1e3, 3),
                          "host_numpy_ms": round(host[k] * 1e3, 1), "host_pairs_timed": len(sub), "card": card}))


if __name__ == "__main__":
    main()
