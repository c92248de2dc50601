"""Benchmark of the GT-annotation pass (gt_info.py): a seeded train_pbr-like split, 640x480, ~15 instances per image,
dense meshes (~50 k faces) in front of and behind a tilted sensor plane.  Reports
  * the GPU pass per instance (device events): renders at both canvases plus the annotation kernel, and the kernel alone;
  * end to end (host clock after a synchronise): images/s and instances/s of run_split, with the JSON and PNG writes;
  * the host PNG encoding of one batch's masks, serially, per mask;
  * a host arm: the numpy restatement of the scripts' per-instance math (gt_info.host_annotation) on the same renders,
    on a subset.
The card's name and power limit are read in the same run.  Prints one JSON line.

  python bench_gt_info.py --images 64 --out /tmp/bench_gt_info.json
"""
import argparse
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from gdrnpp_bop2022_b200 import _lib, bop_eval, gt_info
from gdrnpp_bop2022_b200.ply import save_ply


def uv_ellipsoid(radii, n_lat=160, n_lon=160):
    """A closed ellipsoid mesh (mm) with 2 * n_lon * (n_lat - 1) faces."""
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 0, 1]], v, [[0, 0, -1]]]) * np.asarray(radii)
    idx = lambda i, j: 1 + i * n_lon + (j % n_lon)  # noqa: E731
    f = []
    for j in range(n_lon):
        f.append([0, idx(0, j), idx(0, j + 1)])
        f.append([len(v) - 1, idx(n_lat - 2, j + 1), idx(n_lat - 2, j)])
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f.append([idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)])
            f.append([idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)])
    return v.astype(np.float32), np.asarray(f, np.int32)


def write_tree(root, n_images, per_image, n_objs=8, H=480, W=640, seed=0):
    import cv2

    rs = np.random.RandomState(seed)
    base = os.path.join(root, "lmo")
    os.makedirs(os.path.join(base, "models"))
    n_faces = 0
    for o in range(1, n_objs + 1):
        v, f = uv_ellipsoid(rs.uniform(25, 70, 3))
        save_ply(os.path.join(base, "models", "obj_{:06d}.ply".format(o)), v, f)
        n_faces = len(f)
    per_scene = 25
    for s in range((n_images + per_scene - 1) // per_scene):
        sdir = os.path.join(base, "train_pbr", "{:06d}".format(s))
        os.makedirs(os.path.join(sdir, "depth"))
        gts, cams = {}, {}
        for im in range(min(per_scene, n_images - s * per_scene)):
            K = [572.4, 0.0, 325.3, 0.0, 573.6, 242.0, 0.0, 0.0, 1.0]
            cams[str(im)] = {"cam_K": K, "depth_scale": 0.1}
            yy, xx = np.mgrid[0:H, 0:W]
            mm = 800 + 400 * xx / W + 100 * yy / H + rs.uniform(0, 5, (H, W))
            mm[rs.rand(H, W) < 0.03] = 0
            cv2.imwrite(os.path.join(sdir, "depth", "{:06d}.png".format(im)), np.round(mm / 0.1).astype(np.uint16))
            gts[str(im)] = []
            for _ in range(per_image):
                R = cv2.Rodrigues(rs.uniform(-2, 2, 3))[0]
                z = rs.uniform(600, 1400)
                t = [rs.uniform(-0.45, 0.45) * z, rs.uniform(-0.35, 0.35) * z, z]
                gts[str(im)].append({"obj_id": int(rs.randint(1, n_objs + 1)), "cam_R_m2c": R.ravel().tolist(),
                                     "cam_t_m2c": t})
        for name, c in (("scene_gt.json", gts), ("scene_camera.json", cams)):
            with open(os.path.join(sdir, name), "w") as fh:
                json.dump(c, fh)
    return n_faces


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers still stand; say that the card was not read
        return "not read ({})".format(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--per_image", type=int, default=15)
    ap.add_argument("--batch_images", type=int, default=16)
    ap.add_argument("--host_subset", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gt_info needs a GPU"
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info()}
    with tempfile.TemporaryDirectory() as tmp:
        res["faces_per_mesh"] = write_tree(tmp, a.images, a.per_image)
        sp = gt_info.split_params(tmp, "lmo", "train", "pbr")
        model_dir = gt_info.models_path(tmp, "lmo")
        scenes = gt_info.plan_split(sp)
        ims = scenes[0][1][:a.batch_images]
        meshes = bop_eval.VsdMeshes(gt_info.load_models(model_dir, range(1, 9)), device=dev)
        depth = np.stack([gt_info.read_depth(im["depth"]) for im in ims])
        gts = [(j, g) for j, im in enumerate(ims) for g in im["gts"]]
        args = (meshes, [g["obj_id"] for _, g in gts], np.stack([g["cam_R_m2c"] for _, g in gts]),
                np.stack([np.ravel(g["cam_t_m2c"]) for _, g in gts]), [j for j, _ in gts], np.stack([im["K"] for im in ims]))
        d_depth = torch.from_numpy(depth.view(np.int16)).to(dev)
        scale = [im["depth_scale"] for im in ims]
        n = len(gts)
        H, W = depth.shape[1:]
        # --- GPU pass of one batch: renders + kernel, info and masks ---
        for _ in range(2):
            gt_info.annotate_device(*args, d_depth, scale, masks=True)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gt_info.annotate_device(*args, d_depth, scale, masks=True)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        res["gpu_pass_ms_per_instance"] = [round(t / n, 4) for t in sorted(times)]
        # the kernel alone, on the same renders
        large, small = (torch.stack(x) for x in zip(*[_renders(meshes, args, i, H, W) for i in range(n)]))
        L = _lib.lib()
        counts = torch.empty((n, 3), dtype=torch.int64, device=dev)
        boxes = torch.empty((n, 8), dtype=torch.int32, device=dev)
        masks = torch.empty((2, n, H, W), dtype=torch.uint8, device=dev)
        Ks = torch.from_numpy(np.asarray(args[5], np.float64)).to(dev)
        sc = torch.tensor(scale, dtype=torch.float32, device=dev)
        img = torch.tensor(args[4], dtype=torch.int32, device=dev)

        def kernel():
            _lib.check(L.gdrn_gt_info(_lib.ptr(large), _lib.ptr(small), _lib.ptr(d_depth), _lib.ptr(sc), _lib.ptr(Ks),
                                      _lib.ptr(img), n, H, W, 15.0, _lib.ptr(counts), _lib.ptr(boxes), _lib.ptr(masks[0]),
                                      _lib.ptr(masks[1]), _lib.current_stream()), "gdrn_gt_info")

        kernel()
        torch.cuda.synchronize()
        ktimes = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                kernel()
            e1.record()
            e1.synchronize()
            ktimes.append(e0.elapsed_time(e1) / 10)
        res["kernel_ms_per_instance"] = [round(t / n, 5) for t in sorted(ktimes)]
        kbytes = n * (9 * H * W * 4 + H * W * (4 + 2 + 2)) + len(ims) * H * W * 2   # canvas + image render + masks + sensor
        res["kernel_gb_per_s"] = round(kbytes / (min(ktimes) * 1e-3) / 1e9, 1)
        # host PNG encoding of this batch's masks, serially
        import cv2

        m = masks.cpu().numpy()
        t0 = time.perf_counter()
        for i in range(n):
            for k in range(2):
                cv2.imencode(".png", m[k, i], [cv2.IMWRITE_PNG_COMPRESSION, 3])
        res["png_encode_ms_per_mask"] = round((time.perf_counter() - t0) * 1e3 / (2 * n), 4)
        # host arm: the numpy restatement on the same renders
        ln, sn = large[:a.host_subset].cpu().numpy(), small[:a.host_subset].cpu().numpy()
        t0 = time.perf_counter()
        for i in range(min(a.host_subset, n)):
            j = args[4][i]
            dmm = depth[j].astype(np.float32)
            dmm *= np.float32(scale[j])
            gt_info.host_annotation(ln[i], sn[i], dmm, np.asarray(args[5][j]), 15)
        res["host_numpy_ms_per_instance"] = round((time.perf_counter() - t0) * 1e3 / min(a.host_subset, n), 2)
        # --- end to end: run_split over the whole split (a first run warms the renders and the pools) ---
        gt_info.run_split(sp, model_dir, batch_images=a.batch_images, device=dev, meshes=meshes)
        torch.cuda.synchronize()
        e2e = []
        for _ in range(2):
            t0 = time.perf_counter()
            r = gt_info.run_split(sp, model_dir, batch_images=a.batch_images, device=dev, meshes=meshes)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            e2e.append((r["images"] / dt, r["instances"] / dt))
        res["e2e_images_per_s"] = [round(x[0], 1) for x in e2e]
        res["e2e_instances_per_s"] = [round(x[1], 1) for x in e2e]
        r = None
        for what in (("info",), ("masks",)):
            t0 = time.perf_counter()
            r = gt_info.run_split(sp, model_dir, what=what, batch_images=a.batch_images, device=dev, meshes=meshes)
            torch.cuda.synchronize()
            res["e2e_images_per_s_" + what[0]] = round(r["images"] / (time.perf_counter() - t0), 1)
        res.update({"images": a.images, "instances": r["instances"], "H": int(H), "W": int(W), "batch_images": a.batch_images})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


def _renders(meshes, args, i, H, W):
    from gdrnpp_bop2022_b200 import renderer

    m, obj, R, t, img, K = args
    dev = meshes.device
    ids = torch.tensor([meshes.ids[int(obj[i])]], dtype=torch.int32, device=dev)
    pose = torch.from_numpy(np.concatenate([R[i], t[i].reshape(3, 1)], 1)[None]).to(dev)
    Ki = np.asarray(K[img[i]], np.float64).reshape(1, 3, 3)
    KL = Ki.copy()
    KL[:, 0, 2] += W
    KL[:, 1, 2] += H
    large = renderer.render_meshes(ids, pose, torch.from_numpy(KL).to(dev), 3 * H, 3 * W, bop_eval.VSD_ZNEAR,
                                   bop_eval.VSD_ZFAR)[0]
    small = renderer.render_meshes(ids, pose, torch.from_numpy(Ki).to(dev), H, W, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR)[0]
    return large, small


if __name__ == "__main__":
    main()
