"""EGLRenderer.render benchmark: 1, 8 and 32 instances of a ~30 k-triangle textured mesh at 640 x 480.

  scene_all_ms   render(image_tensor=, seg_tensor=, normal_tensor=, pc_obj_tensor=, pc_cam_tensor=): one
                 rast_render_scene launch set plus the copies into the [H,W,4] tensors
  scene_pc_ms    render(pc_cam_tensor=) alone
  loop_pc_ms     the per-instance loop EGLRenderer.render ran before the scene render (one render_depth per instance,
                 then a torch.where composite), pc_cam only

Each entry is [median, 10th percentile, 90th percentile] of the CUDA-event milliseconds per call over --iters calls
after --warmup, then the median host milliseconds to issue the call: when that is close to the event time, the call
is bound by the host's launches, not by the GPU.  Prints one JSON line; writes nothing to disk.

  python bench_render.py [--iters 50] [--warmup 10]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from gdrnpp_bop2022_b200.renderer import EGLRenderer, Model3D, render_depth
from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

H, W = 480, 640
K = np.array([[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]], np.float32)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown ({})".format(e)


def textured_mesh(dev):
    """Icosphere subdivided to 20480 triangles plus a 10 k-triangle band of it again, so ~30 k triangles, with
    spherical UVs and a 1024 x 1024 texture."""
    v, f = make_icosphere_mesh(5, (0.12, 0.08, 0.1))
    v = np.asarray(v, np.float32)
    f = np.asarray(f, np.int32)
    f = np.concatenate([f, f[: len(f) // 2][:, [0, 2, 1]]])
    d = v / np.linalg.norm(v, axis=1, keepdims=True)
    uv = np.stack([0.5 + np.arctan2(d[:, 1], d[:, 0]) / (2 * np.pi), np.arccos(np.clip(d[:, 2], -1, 1)) / np.pi], 1)
    y, x = np.mgrid[0:1024, 0:1024]
    tex = np.stack([x % 256, y % 256, (x ^ y) % 256], -1).astype(np.uint8)
    return Model3D(v, f, device=dev, normals=d, uvs=uv.astype(np.float32), texture=tex)


def poses(n, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        q, r = np.linalg.qr(rs.randn(3, 3))
        q = q * np.sign(np.diag(r))
        q[:, 0] *= np.linalg.det(q)
        t = [rs.uniform(-0.15, 0.15), rs.uniform(-0.1, 0.1), rs.uniform(0.6, 1.2)]
        out.append(np.hstack([q, np.array(t)[:, None]]).astype(np.float32))
    return out


def old_loop(model, ps, dev):
    Kt = torch.from_numpy(K)[None].to(dev)
    depth = torch.zeros((H, W), device=dev)
    xyz = torch.zeros((H, W, 3), device=dev)
    for p in ps:
        d, x = render_depth(model, torch.from_numpy(p)[None].to(dev), Kt, H, W, 0.25, 6.0, return_xyz=True)
        upd = (d[0] > 0) & ((depth == 0) | (d[0] < depth))
        depth = torch.where(upd, d[0], depth)
        xyz = torch.where(upd[..., None], x[0], xyz)
    return depth, xyz


def timed(fn, iters, warmup):
    """-> (median, p10, p90) of the CUDA-event time and the median host time to issue the call, all in ms."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts, hs = [], []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        h0 = time.perf_counter()
        fn()
        hs.append((time.perf_counter() - h0) * 1e3)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return [round(float(x), 4) for x in (np.median(ts), np.percentile(ts, 10), np.percentile(ts, 90), np.median(hs))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_render.py needs a GPU"
    dev = torch.device("cuda:0")
    model = textured_mesh(dev)
    egl = EGLRenderer([model], K=K, width=W, height=H, device=dev)
    bufs = {k: torch.zeros((H, W, 4), device=dev) for k in ("image", "seg", "normal", "pc_obj", "pc_cam")}
    out = {"gpu": gpu_info(), "triangles": int(model.faces.shape[0]), "H": H, "W": W, "cases": []}
    for n in (1, 8, 32):
        ps = poses(n, seed=n)
        ids = [0] * n
        all_ms = timed(lambda: egl.render(ids, ps, image_tensor=bufs["image"], seg_tensor=bufs["seg"],
                                          normal_tensor=bufs["normal"], pc_obj_tensor=bufs["pc_obj"],
                                          pc_cam_tensor=bufs["pc_cam"]), a.iters, a.warmup)
        pc_ms = timed(lambda: egl.render(ids, ps, pc_cam_tensor=bufs["pc_cam"]), a.iters, a.warmup)
        loop_ms = timed(lambda: old_loop(model, ps, dev), a.iters, a.warmup)
        out["cases"].append({"instances": n, "scene_all_ms": all_ms, "scene_pc_ms": pc_ms, "loop_pc_ms": loop_ms})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
