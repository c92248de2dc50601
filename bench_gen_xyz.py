"""Benchmark of the xyz_crop generator (gen_xyz.py): a seeded train_pbr-like split of 720x540 images, ~15 instances per
image of 10 icosphere meshes of ~20 k faces at 0.4 - 1.5 m, a few of them off the frame.  Reports
  * the GPU pass (device events around gen_xyz.crops_async on one batch of images): renders, boxes, one boxes read-back,
    pack and the crops' copy, in instances/s;
  * end to end (host clock): run_split over the whole split into a temporary directory, pickles included, in
    instances/s;
  * the per-instance arm on a subset, the reference loop's shape on this repository's renderer: per instance
    EGLRenderer.render([i], [pose], K=, seg_tensor=, pc_cam_tensor=), the box from the mask with four .item() syncs,
    misc.calc_xyz_bp_torch restated in torch, .cpu() of the crop and the pickle, in instances/s.
Every figure is listed over its repeats, sorted (the spread).  The card's name and power limit are read in the same run.
Prints one JSON line.

  python bench_gen_xyz.py --images 240 --out /tmp/bench_gen_xyz.json
"""
import argparse
import json
import os
import pickle
import shutil
import tempfile
import time

import numpy as np
import torch

from bench_gt_info import gpu_info
from gdrnpp_bop2022_b200 import gen_xyz, gt_info
from gdrnpp_bop2022_b200.ply import save_ply
from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh


def write_tree(root, n_images, per_image, n_objs=10, H=540, W=720, per_scene=50, seed=0):
    """BOP_DATASETS/tless/{models_cad, train_pbr}: rgb/*.jpg (for the image size), scene_gt.json, scene_camera.json."""
    import cv2

    rs = np.random.RandomState(seed)
    base = os.path.join(root, "BOP_DATASETS", "tless")
    os.makedirs(os.path.join(base, "models_cad"))
    n_faces = 0
    for o in range(1, n_objs + 1):
        v, f = make_icosphere_mesh(5, rs.uniform(60, 200, 3))
        save_ply(os.path.join(base, "models_cad", "obj_{:06d}.ply".format(o)), v, f)
        n_faces = len(f)
    img = cv2.GaussianBlur(rs.randint(0, 256, (H, W, 3)).astype(np.uint8), (7, 7), 2.0)
    n_off = 0
    for s in range((n_images + per_scene - 1) // per_scene):
        sdir = os.path.join(base, "train_pbr", "{:06d}".format(s))
        os.makedirs(os.path.join(sdir, "rgb"))
        gts, cams = {}, {}
        for im in range(min(per_scene, n_images - s * per_scene)):
            f = 1075.0 * rs.uniform(0.95, 1.05)
            cams[str(im)] = {"cam_K": [f, 0.0, W / 2 + rs.uniform(-3, 3), 0.0, f, H / 2 + rs.uniform(-3, 3), 0.0, 0.0, 1.0],
                             "depth_scale": 0.1}
            cv2.imwrite(os.path.join(sdir, "rgb", "{:06d}.jpg".format(im)), img)
            gts[str(im)] = []
            for k in range(per_image):
                R = cv2.Rodrigues(rs.uniform(-2, 2, 3))[0]
                z = rs.uniform(400, 1500)
                t = [rs.uniform(-0.3, 0.3) * z, rs.uniform(-0.22, 0.22) * z, z]
                if k == 0 and im % 8 == 0:   # a few instances off the frame
                    t[0] = 3 * z
                    n_off += 1
                gts[str(im)].append({"obj_id": int(rs.randint(1, n_objs + 1)), "cam_R_m2c": R.ravel().tolist(),
                                     "cam_t_m2c": t})
        for name, c in (("scene_gt.json", gts), ("scene_camera.json", cams)):
            with open(os.path.join(sdir, name), "w") as fh:
                json.dump(c, fh)
    return n_faces, n_off


def calc_xyz_bp_torch(depth, R, T, K):
    """misc.calc_xyz_bp_torch (lib/pysixd/misc.py), restated."""
    height, width = depth.shape
    mask = (depth != 0).to(depth).view(height, width, 1)
    grid_y, grid_x = torch.meshgrid(torch.arange(height, device=depth.device, dtype=depth.dtype) - K[1, 2],
                                    torch.arange(width, device=depth.device, dtype=depth.dtype) - K[0, 2], indexing="ij")
    xyz_cam = torch.stack((grid_x * depth / K[0, 0], grid_y * depth / K[1, 1], depth), dim=2).view(height, width, 3, 1)
    Rinv = R.t().view(1, 1, 3, 3).expand(height, width, 3, 3)
    T_expand = T.view(1, 1, 3, 1).expand(height, width, 3, 1)
    return torch.einsum("hwij,hwjk->hwi", Rinv, xyz_cam - T_expand) * mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=240)
    ap.add_argument("--per_image", type=int, default=15)
    ap.add_argument("--batch_images", type=int, default=16)
    ap.add_argument("--subset", type=int, default=120, help="instances of the per-instance arm")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gen_xyz needs a GPU"
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info()}
    with tempfile.TemporaryDirectory() as tmp:
        res["faces_per_mesh"], res["off_frame_instances"] = write_tree(tmp, a.images, a.per_image)
        bop = os.path.join(tmp, "BOP_DATASETS")
        sp = gt_info.split_params(bop, "tless", "train", "pbr")
        model_dir = gt_info.models_path(bop, "tless")
        xyz_root = os.path.join(tmp, "xyz_crop")
        scenes, _ = gen_xyz.plan(sp, xyz_root)
        scene_id, (H, W), todo, _ = scenes[0]
        insts = [i for _, ii in todo[:a.batch_images] for i in ii]
        models = gen_xyz.load_models(model_dir, range(1, 11), device=dev)
        order = sorted(models)
        mlist = [models[o] for o in order]
        args = (mlist, [order.index(i["obj_id"]) for i in insts], np.stack([i["R"] for i in insts]),
                np.stack([i["t"] for i in insts]), np.stack([i["K"] for i in insts]), H, W)
        n = len(insts)
        # --- GPU pass of one batch ---
        staging = gt_info._Staging()
        for _ in range(2):
            gen_xyz.crops_async(*args, staging=staging)[-1].synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = gen_xyz.crops_async(*args, staging=staging)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        res["gpu_pass_instances_per_s"] = [round(n / (t * 1e-3), 1) for t in sorted(times, reverse=True)]
        res["batch_instances"] = n
        res["crop_bytes_per_batch"] = int(out[2][-1]) * 2
        # --- end to end: run_split over the whole split (a first run warms the pools and the allocator) ---
        e2e = []
        for rep in range(1 + min(a.reps, 3)):
            shutil.rmtree(xyz_root, ignore_errors=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = gen_xyz.run_split(sp, model_dir, xyz_root, batch_images=a.batch_images, device=dev, log=None,
                                  models=models)
            torch.cuda.synchronize()
            if rep:
                e2e.append(r["written"] / (time.perf_counter() - t0))
        res["e2e_instances_per_s"] = [round(x, 1) for x in sorted(e2e)]
        res.update({"images": r["images"], "instances": r["written"], "empty_instances": r["empty"]})
        # --- the per-instance arm: the reference loop's shape on EGLRenderer.render ---
        from gdrnpp_bop2022_b200 import renderer

        egl = renderer.EGLRenderer(mlist, height=H, width=W, znear=gen_xyz.ZNEAR, zfar=gen_xyz.ZFAR, device=dev)
        seg = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        pc_cam = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        sub = insts[:a.subset]
        arm_dir = os.path.join(tmp, "arm")
        os.makedirs(arm_dir)

        def one(k, inst):
            pose = np.hstack([inst["R"], inst["t"].reshape(3, 1)])
            egl.render([order.index(inst["obj_id"])], [pose], K=inst["K"], seg_tensor=seg, pc_cam_tensor=pc_cam)
            mask = (seg[:, :, 0] > 0).to(torch.uint8)
            if mask.sum() == 0:
                info = {"xyz_crop": np.zeros((H, W, 3), dtype=np.float16), "xyxy": [0, 0, W - 1, H - 1]}
            else:
                ys_xs = mask.nonzero(as_tuple=False)
                ys, xs = ys_xs[:, 0], ys_xs[:, 1]
                x1, y1 = [xs.min().item(), ys.min().item()]
                x2, y2 = [xs.max().item(), ys.max().item()]
                xyz = calc_xyz_bp_torch(pc_cam[:, :, 2], torch.tensor(inst["R"], device=dev),
                                        torch.tensor(inst["t"], device=dev), torch.tensor(inst["K"], device=dev))
                info = {"xyz_crop": xyz[y1:y2 + 1, x1:x2 + 1].cpu().numpy().astype("float16"), "xyxy": [x1, y1, x2, y2]}
            with open(os.path.join(arm_dir, "{}.pkl".format(k)), "wb") as f:
                pickle.dump(info, f, protocol=2)

        for k, inst in enumerate(sub[:8]):
            one(k, inst)
        arm = []
        for _ in range(min(a.reps, 3)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for k, inst in enumerate(sub):
                one(k, inst)
            torch.cuda.synchronize()
            arm.append(len(sub) / (time.perf_counter() - t0))
        res["per_instance_arm_instances_per_s"] = [round(x, 1) for x in sorted(arm)]
        res["per_instance_arm_instances"] = len(sub)
        res.update({"H": int(H), "W": int(W), "batch_images": a.batch_images})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
