#!/usr/bin/env python
"""bench_postprocess.py -- the test-time post-processes on one H100: every TEST.PNP_TYPE (ransac_pnp and the three
network-initialised types) and both fast-depth-refine weightings (||xyz|| and TEST.USE_COOR_Z_REFINE), at B = 5 and
B = 64 ROIs of 64x64 maps.

  python bench_postprocess.py [--reps 50] [--warmup 5] [--host-reps 3]

For each case it times the batched GPU call with CUDA events after warm-up (median ms per batch), and the reference's
per-ROI host loop on the same maps (median wall ms per batch): get_out_mask + correspondence selection + the cv2 call
of gdrn_evaluator.py:241-371 / 1122-1221 for PnP, the numpy weighting / median / ray of gdrn_evaluator.py:528-561 for
one refine iteration (the GPU side of that row is one refine step on the same rendered depth).  Prints one JSON line
per case plus the card's name and power limit, read in the same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_per_object import card_info  # noqa: E402

K_CAM = np.array([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]])


def make_maps(B, seed, hw=64, imH=480, imW=640):
    """Noisy coordinate / mask maps of a sphere-shaped object (r = 5 cm) at 0.7-0.9 m seen through each ROI grid, with
    a network pose 2 deg / 1 cm off the truth."""
    import cv2

    rs = np.random.RandomState(seed)
    out = {k: [] for k in ("cx", "cy", "cz", "m", "c2d", "ext", "R", "t")}
    for _ in range(B):
        ax = rs.randn(3)
        ang = rs.rand() * 3
        R = cv2.Rodrigues(ax / np.linalg.norm(ax) * ang)[0]
        t = np.array([rs.randn() * 0.05, rs.randn() * 0.05, 0.7 + rs.rand() * 0.2])
        e = np.array([0.12, 0.13, 0.11])
        pc = K_CAM @ t
        pc = pc[:2] / pc[2]
        scale = 2.6 * 0.05 * K_CAM[0, 0] / t[2]
        U, V = np.meshgrid(pc[0] + (np.arange(hw) - hw / 2) * scale / hw, pc[1] + (np.arange(hw) - hw / 2) * scale / hw)
        rays = np.stack([(U - K_CAM[0, 2]) / K_CAM[0, 0], (V - K_CAM[1, 2]) / K_CAM[1, 1], np.ones_like(U)], -1)
        rays /= np.linalg.norm(rays, axis=-1, keepdims=True)
        b_ = (rays * t).sum(-1)
        disc = b_ ** 2 - (t @ t - 0.05 ** 2)
        hit = disc > 0
        Xc = rays * (b_ - np.sqrt(np.where(hit, disc, 0)))[..., None]
        coor = (Xc - t) @ R / e + 0.5 + rs.randn(hw, hw, 3) * 0.002
        coor[~hit] = 0.5
        out["cx"].append(coor[..., 0]); out["cy"].append(coor[..., 1]); out["cz"].append(coor[..., 2])
        out["m"].append(np.where(hit, 0.9, 0.05) + rs.randn(hw, hw) * 0.02)
        out["c2d"].append(np.stack([U / imW, V / imH])); out["ext"].append(e)
        dR = cv2.Rodrigues(rs.randn(3) / np.sqrt(3) * np.deg2rad(2))[0]
        out["R"].append(dR @ R); out["t"].append(t + rs.randn(3) * 0.01)
    d = {k: np.stack(v).astype(np.float32) for k, v in out.items()}
    d.update(imH=imH, imW=imW)
    return d


def host_pnp(d, pnp_type):
    """The reference's per-ROI loop: get_out_mask (L1), get_img_model_points_with_coords2d, then the cv2 call."""
    import cv2

    out_transes = d["t"].copy()
    for i in range(d["cx"].shape[0]):
        m = d["m"][i]
        mn = (m - m.min()) / (m.max() - m.min())
        e = d["ext"][i]
        xyz = np.stack([(d["cx"][i] - 0.5) * e[0], (d["cy"][i] - 0.5) * e[1], (d["cz"][i] - 0.5) * e[2]], -1)
        sel = (mn > 0.5) & (np.abs(xyz[..., 0]) > 1e-4 * e[0]) & (np.abs(xyz[..., 1]) > 1e-4 * e[1]) & (np.abs(xyz[..., 2]) > 1e-4 * e[2])
        img = np.stack([d["c2d"][i][0] * d["imW"], d["c2d"][i][1] * d["imH"]], -1)
        p3 = np.ascontiguousarray(xyz[sel].astype(np.float64))
        p2 = np.ascontiguousarray(img[sel].astype(np.float64))
        dist = np.zeros((8, 1))
        if pnp_type == "ransac_pnp":
            cv2.solvePnPRansac(p3[None], p2[None], K_CAM, dist, flags=cv2.SOLVEPNP_EPNP, reprojectionError=3.0, iterationsCount=100)
        elif pnp_type == "net_iter_pnp":
            cv2.solvePnP(p3, p2, K_CAM, dist, rvec=cv2.Rodrigues(d["R"][i])[0], tvec=out_transes[i], useExtrinsicGuess=True,
                         flags=cv2.SOLVEPNP_ITERATIVE)
        else:
            cv2.solvePnPRansac(p3[None], p2[None], K_CAM, dist, flags=cv2.SOLVEPNP_EPNP, useExtrinsicGuess=True,
                               rvec=cv2.Rodrigues(d["R"][i])[0], tvec=out_transes[i], reprojectionError=3.0, iterationsCount=20)


def host_refine_step(xyz01, mask, sensor, ren, Ks, R, t, coor_z):
    """One iteration of gdrn_evaluator.py:528-561 per ROI (the render excluded)."""
    for i in range(mask.shape[0]):
        x = xyz01[i].transpose(1, 2, 0)
        mi = (mask[i] - mask[i].min()) / (mask[i].max() - mask[i].min())
        if coor_z:
            q = (R[i] @ x.reshape(-1, 3).T).T.reshape(64, 64, 3)[:, :, -1] * mi
        else:
            q = np.linalg.norm(x, axis=-1) * mi
        q = q * (ren[i] > 0) * (sensor[i] > 0)
        s = q.sum()
        if s == 0:
            continue
        q /= s
        yy, xx = np.argwhere(q > q.max() * 0.8).T
        dz = np.median(sensor[i][yy, xx] - ren[i][yy, xx])
        yx = np.stack(np.meshgrid(np.arange(64), np.arange(64))[::-1], axis=-1)
        ray = np.linalg.inv(Ks[i]) @ (*(yx * q[..., None]).sum(axis=(0, 1))[::-1], 1)
        t[i] = t[i] + ray / ray[2] * dz


def cuda_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def host_ms(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()
    from gdrnpp_bop2022_b200 import _lib
    from gdrnpp_bop2022_b200.pnp_ransac import pnp_net_from_maps, pnp_ransac_from_maps
    from gdrnpp_bop2022_b200.renderer import Model3D, render_depth
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    dev = torch.device("cuda:0")
    print(json.dumps({"card": card_info(0)}), flush=True)
    for B in (5, 64):
        d = make_maps(B, seed=B)
        T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        maps = (T(d["cx"][:, None]), T(d["cy"][:, None]), T(d["cz"][:, None]), T(d["m"][:, None]), T(d["c2d"]),
                torch.full((B,), float(d["imH"])), torch.full((B,), float(d["imW"])), T(d["ext"]),
                T(np.repeat(K_CAM[None].astype(np.float32), B, 0)))
        R, t = T(d["R"]), T(d["t"])
        for pnp_type in ("ransac_pnp", "net_iter_pnp", "net_ransac_pnp", "net_ransac_pnp_rot"):
            if pnp_type == "ransac_pnp":
                fn = lambda: pnp_ransac_from_maps(*maps)
            else:
                fn = lambda: pnp_net_from_maps(*maps, R, t, pnp_type=pnp_type)
            g = cuda_ms(fn, a.reps, a.warmup)
            h = host_ms(lambda: host_pnp(d, pnp_type), a.host_reps)
            print(json.dumps({"B": B, "case": "pnp", "pnp_type": pnp_type, "gpu_ms": round(g, 4), "host_cv2_ms": round(h, 3),
                              "speedup": round(h / g, 1)}), flush=True)
        # depth refine: one refine step on a rendered depth (the render is common to both weightings)
        v, f = make_icosphere_mesh(3, (0.1, 0.1, 0.1))
        rs = np.random.RandomState(B)
        Kc = np.stack([np.array([[110.0 + 10 * rs.rand(), 0, 32], [0, 112.0, 31], [0, 0, 1]]) for _ in range(B)]).astype(np.float32)
        poses = torch.cat([R, t[:, :, None]], 2).contiguous()
        ren = render_depth(Model3D(v, f, device=dev), poses, T(Kc), 64, 64)
        sensor = (ren * 1.02).contiguous()
        xyz = T(np.concatenate([d["cx"][:, None], d["cy"][:, None], d["cz"][:, None]], 1))
        mask = T(d["m"])
        ren_h, sen_h, xyz_h, mask_h = ren.cpu().numpy(), sensor.cpu().numpy(), xyz.cpu().numpy(), d["m"]
        Kd = T(Kc)
        for coor_z in (False, True):
            tt = t.clone()

            def step():
                _lib.check(_lib.lib().gdrn_depth_refine_step(_lib.ptr(xyz), _lib.ptr(mask), 1, _lib.ptr(sensor), _lib.ptr(ren),
                                                             _lib.ptr(Kd), _lib.ptr(R), int(coor_z), _lib.ptr(tt), B, 64, 0.8,
                                                             _lib.current_stream()), "gdrn_depth_refine_step")
            g = cuda_ms(step, a.reps, a.warmup)
            th = d["t"].astype(np.float64).copy()
            h = host_ms(lambda: host_refine_step(xyz_h, mask_h, sen_h, ren_h, Kc.astype(np.float64), d["R"], th, coor_z), a.host_reps)
            print(json.dumps({"B": B, "case": "depth_refine_step", "weighting": "coor_z" if coor_z else "norm_xyz", "gpu_ms": round(g, 4),
                              "host_numpy_ms": round(h, 3), "speedup": round(h / g, 1)}), flush=True)


if __name__ == "__main__":
    main()
