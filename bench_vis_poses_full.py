"""Pose outline benchmark (vis_poses_full): on a synthetic split at 640 x 480 and 1280 x 960 with 6 and 20 instances per
image (every GT instance kept, one estimate per GT instance), times
  * the device pass per image (gdrn_vis_gray3, rast_render_scene_bg, rast_render_meshes and gdrn_vis_outlines on
    staged inputs, CUDA events),
  * the driver end to end (vis_poses_full.run_split with the models loaded: decode, passes, PNG writes),
  * the scripts' loop on this repository's renderer: one EGLRenderer.render and one D2H copy per instance, NumPy
    get_edge and painting (oracle/vis_poses_full_oracle.py),
and checks that the device pass and the scripts' loop give equal composites.  Prints one JSON line with the card's name
and power limit; writes only under a temporary directory.

  python bench_vis_poses_full.py [--images 8] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gdrnpp_bop2022_b200 import gt_info  # noqa: E402
from gdrnpp_bop2022_b200 import vis_poses as VP  # noqa: E402
from gdrnpp_bop2022_b200 import vis_poses_full as VF  # noqa: E402
from gdrnpp_bop2022_b200.renderer import EGLRenderer  # noqa: E402
from gdrnpp_bop2022_b200.synthetic import write_bop_tree  # noqa: E402
from oracle import vis_poses_full_oracle as O  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "unknown ({})".format(e)


def one_config(tmp, H, W, inst, n_images, iters, dev):
    root = os.path.join(tmp, "d{}x{}_{}".format(W, H, inst))
    write_bop_tree(root, dataset="ycbv", num_images=n_images, num_scenes=1, H=H, W=W, dets_per_image=inst,
                   obj_ids=list(range(1, 21)))
    sp = gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "ycbv", "test")
    rs = np.random.RandomState(0)
    results = {}
    for im in VP.plan_images(sp):
        results[(im[0], im[1])] = [{"obj_id": int(p["obj_id"]), "score": 0.9,
                                    "R": np.asarray(p["R"]).reshape(3, 3) @ cv2.Rodrigues(rs.uniform(-0.2, 0.2, 3))[0],
                                    "t": (np.asarray(p["t"], np.float64).ravel() + rs.uniform(-15, 15, 3)) / 1000}
                                   for p in im[6]]
    models_dir = os.path.join(sp["base_path"], "models_eval")
    images = VF.plan(sp, results=results)
    used = sorted({p["obj_id"] for im in images for p in im[6]})
    models = VF.load_models(models_dir, used, dev)
    n_inst = sum(len(im[6]) for im in images)

    # device pass on staged inputs
    rgb = np.stack([VP.read_rgb(im[5]) for im in images])
    d_rgb = torch.from_numpy(rgb).to(dev)
    Ks = np.stack([im[2] for im in images])
    out = torch.empty((len(images), H, W, 3), dtype=torch.uint8, device=dev)

    def device_pass():
        VF.render_batch(models, images, VF.gray3(d_rgb), Ks, H, W, out)

    device_pass()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        device_pass()
    e1.record()
    torch.cuda.synchronize()
    dev_ms = e0.elapsed_time(e1) / iters / len(images)
    got = out.cpu().numpy()

    # the scripts' loop on this repository's renderer
    ren = EGLRenderer(list(models.values()), model_ids=list(models), width=W, height=H, device=dev)
    image_tensor = torch.empty((H, W, 4), device=dev)
    seg_tensor = torch.empty((H, W, 4), device=dev)
    equal = True
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for j, im in enumerate(images):
        est = [p for p in im[6] if not p["gt"]]
        gray = O.bgr2gray3(rgb[j][..., ::-1])
        ren.render([p["obj_id"] for p in est], [np.hstack([p["R"], p["t"].reshape(3, 1)]) for p in est], K=im[2],
                   image_tensor=image_tensor, background=gray)
        ren_bgr = (image_tensor[:, :, :3].cpu().numpy() + 0.5).astype("uint8")
        for gt_pass, col in ((True, (255, 0, 0)), (False, (0, 255, 0))):
            for p in im[6]:
                if p["gt"] != gt_pass:
                    continue
                ren.render([p["obj_id"]], [np.hstack([p["R"], p["t"].reshape(3, 1)])], K=im[2], seg_tensor=seg_tensor)
                ren_bgr[O.get_edge((seg_tensor[:, :, 0].cpu().numpy() > 0).astype("uint8"), 3)] = col
        equal = equal and np.array_equal(ren_bgr, got[j])
    host_ms = 1e3 * (time.perf_counter() - t0) / len(images)

    vis = os.path.join(tmp, "vis{}x{}_{}".format(W, H, inst))
    VF.run_split(sp, models_dir, vis, results, device=dev, models=models)   # warm-up
    r = VF.run_split(sp, models_dir, vis, results, device=dev, models=models)
    return {"H": H, "W": W, "instances_per_image": n_inst / len(images), "images": len(images),
            "device_pass_ms_per_image": dev_ms, "device_pass_images_per_s": 1e3 / dev_ms,
            "run_split_images_per_s": r["images"] / r["seconds"], "scripts_loop_ms_per_image": host_ms,
            "scripts_loop_images_per_s": 1e3 / host_ms, "outputs_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vis_poses_full.py needs a GPU"
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "configs": []}
    with tempfile.TemporaryDirectory() as tmp:
        for H, W in ((480, 640), (960, 1280)):
            for inst in (6, 20):
                res["configs"].append(one_config(tmp, H, W, inst, a.images, a.iters, dev))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
