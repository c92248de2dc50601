"""Pose visualisation benchmark: the GPU pass per image (flat-shaded renders + composite, device inputs staged before
the timed window), the split driver end to end on a synthetic split (vis_poses.run_split, the CLI's loop, with the
meshes already uploaded and after one warm-up pass), and the host arm (the reference's NumPy compositing, restated in vis_poses.host_vis_object_poses,
run on the same renders).  The reference's GL renders cannot be timed without a GL context and are not measured.
Prints one JSON line; writes only under a temporary directory.

  python bench_vis_poses.py [--images 32] [--inst 8] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import torch

from gdrnpp_bop2022_b200 import bop_eval, gt_info
from gdrnpp_bop2022_b200 import vis_poses as VP
from gdrnpp_bop2022_b200.ply import load_ply
from gdrnpp_bop2022_b200.synthetic import write_bop_tree


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown ({})".format(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--inst", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vis_poses.py needs a GPU"
    dev = torch.device("cuda:0")
    out = {"gpu": gpu_info()}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "datasets")
        write_bop_tree(root, dataset="ycbv", num_images=a.images, num_scenes=2, H=480, W=640, dets_per_image=a.inst,
                       obj_ids=list(range(1, 9)))
        sp = gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "ycbv", "test")
        images = VP.plan_images(sp)
        used = sorted({int(p["obj_id"]) for im in images for p in im[6]})
        ms = {o: load_ply(os.path.join(sp["base_path"], "models_eval", "obj_{:06d}.ply".format(o))) for o in used}
        meshes = bop_eval.VsdMeshes({o: (m["pts"], m["faces"]) for o, m in ms.items()}, device=dev)
        pal = VP.default_colors()
        oc = {o: tuple(pal[(o - 1) % len(pal)]) for o in used}
        ppi = [im[6] for im in images]
        K = np.stack([im[2] for im in images])
        rgb = np.stack([VP.read_rgb(im[5]) for im in images])
        depth = np.stack([gt_info.read_depth(im[4]).astype(np.float32) * np.float32(im[3]) for im in images])
        d_rgb, d_depth = torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev)
        n_inst = sum(len(p) for p in ppi)
        flags = VP.RGB | VP.RESOLVE | VP.DEPTH_DIFF

        # the device inputs are staged once, so the timed window holds the launches only
        from gdrnpp_bop2022_b200 import renderer

        inst = [(j, p) for j, ps in enumerate(ppi) for p in ps]
        ids = torch.tensor([meshes.ids[int(p["obj_id"])] for _, p in inst], dtype=torch.int32, device=dev)
        poses = torch.from_numpy(np.concatenate([np.stack([np.asarray(p["R"], np.float64).reshape(3, 3) for _, p in inst]),
                                                 np.stack([np.asarray(p["t"], np.float64).reshape(3, 1) for _, p in inst])],
                                                axis=2)).float().to(dev)
        Ks = torch.from_numpy(K[[j for j, _ in inst]]).float().to(dev)
        cols = torch.tensor([oc[int(p["obj_id"])] for _, p in inst], dtype=torch.float32, device=dev)
        off = np.cumsum([0] + [len(p) for p in ppi])
        off_dev = torch.from_numpy(off.astype(np.int32)).to(dev)

        def gpu_pass():
            m_rgb, m_depth = renderer.render_meshes_rgb(ids, poses, Ks, 480, 640, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR,
                                                        colors=cols)
            return VP.composite_device(m_rgb, m_depth, off, d_rgb, d_depth, flags, inst_off_dev=off_dev), m_rgb, m_depth

        for _ in range(3):
            gpu_pass()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            gpu_pass()
        e1.record()
        torch.cuda.synchronize()
        ms_pass = e0.elapsed_time(e1) / a.iters
        out.update({"images": len(images), "instances": n_inst, "H": 480, "W": 640,
                    "gpu_pass_ms_per_image": ms_pass / len(images), "gpu_pass_us_per_instance": 1e3 * ms_pass / n_inst})
        _, m_rgb, m_depth = gpu_pass()
        m_rgb, m_depth = m_rgb.cpu().numpy(), m_depth.cpu().numpy()
        t0 = time.perf_counter()
        for j in range(len(images)):
            VP.host_vis_object_poses(m_rgb[off[j]:off[j + 1]], m_depth[off[j]:off[j + 1]], rgb[j], depth[j],
                                     [p["text_info"] for p in ppi[j]])
        out["host_numpy_ms_per_image"] = 1e3 * (time.perf_counter() - t0) / len(images)
        vis = os.path.join(tmp, "vis")
        VP.run_split(sp, os.path.join(sp["base_path"], "models_eval"), vis, "ycbv", "test", meshes=meshes)   # warm
        r = VP.run_split(sp, os.path.join(sp["base_path"], "models_eval"), vis, "ycbv", "test", meshes=meshes)
        out["run_split_images_per_s"] = r["images"] / r["seconds"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
