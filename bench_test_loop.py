"""Throughput of the dataset test loop (gdrn_evaluator.gdrn_inference_on_dataset) on a synthetic BOP split.

Writes ~300 images of 640 x 480 (random BGR PNG + 16-bit depth PNG, ~6 detections each, box meshes) into a temporary
directory, loads seeded weights (synthetic.make_state_dict), and prints one JSON line with the card name and power limit:
  * images/s and ROIs/s of the loop at max_batch=64, and with one image per forward (the reference's batch_size=1);
  * the per-stage times of the max_batch=64 run: decode (host seconds summed over the decoder threads, which overlap
    the device), h2d / roi_build / forward / post / d2h (CUDA events), csv (host);
  * GPU time of gdrn_roi_setup + gdrn_roi_crop_multi for one batch against the per-image path it replaces (host
    get_affine_transform per ROI + three crop_resize launches per image), for the same ROIs.
The network runs in bf16x3 with the network pose (no PnP), the BOP test configs' default.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_yolox import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=300)
    ap.add_argument("--precision", default="bf16x3")
    args = ap.parse_args()
    import types

    from gdrnpp_bop2022_b200 import bop_eval
    from gdrnpp_bop2022_b200 import gdrn_evaluator as G
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg
    from gdrnpp_bop2022_b200.native_ops import crop_resize_float, crop_resize_image, get_affine_transform
    from gdrnpp_bop2022_b200.synthetic import make_state_dict, write_bop_tree

    dev = torch.device("cuda:0")
    name = card()
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "datasets")
        det = write_bop_tree(root, num_images=args.images, num_scenes=6, dets_per_image=6, seed=0)
        cfg = default_cfg()
        cfg.VAL = types.SimpleNamespace(DATASET_NAME="ycbv", SPLIT="test", SPLIT_TYPE="", USE_BOP=True,
                                        TARGETS_FILENAME="test_targets_bop19.json")
        cfg.DATASETS = types.SimpleNamespace(DET_FILES_TEST=(det,), DET_THR=0.0, DET_TOPK_PER_OBJ=1)
        model = GDRN_DoubleMask(cfg, max_batch=64, precision=args.precision)
        model.load_state_dict(make_state_dict(num_classes=21, seed=0))
        model.to(dev)
        ts = G.TestSet(cfg, root)
        G.gdrn_inference_on_dataset(cfg, model, root, max_batch=64, test_set=ts)   # warm-up: graphs, page cache
        G.gdrn_inference_on_dataset(cfg, model, root, max_batch=1, test_set=ts)
        res = {}
        for mb in (64, 1):
            stats = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows = G.gdrn_inference_on_dataset(cfg, model, root, max_batch=mb, test_set=ts, stats=stats)
            wall = time.perf_counter() - t0
            res[mb] = (rows, wall, stats)
        rows, wall, stats = res[64]
        t0 = time.perf_counter()
        bop_eval.write_bop_results_csv(rows, os.path.join(tmp, "res.csv"))
        csv_s = time.perf_counter() - t0

        # ROI build of one 64-ROI batch: the two kernels against the per-image path
        from gdrnpp_bop2022_b200.native_ops import roi_batch_inputs

        recs = ts.records
        batch = G.pack_batches([len(a) for _, a in recs], 64)[0]
        imgs = [recs[p] for p in batch]
        ims = [G.read_image(ts.rgb[i]) for i, _ in imgs]
        H, W = ims[0].shape[:2]
        images = torch.from_numpy(np.stack(ims)).to(dev)
        meta = torch.tensor([(j, a["label"]) for j, (_, anns) in enumerate(imgs) for a in anns], dtype=torch.int32, device=dev)
        xywh = torch.tensor([a["bbox_est"] for _, anns in imgs for a in anns], dtype=torch.float32, device=dev)
        Ks = torch.from_numpy(np.stack([ts.K[i] for i, _ in imgs])).to(dev)
        ext = torch.rand((21, 3), device=dev)
        grid = None

        depth = torch.zeros((len(imgs), H, W), dtype=torch.uint16, device=dev)
        factor = torch.ones((len(imgs),), dtype=torch.float64, device=dev)

        def batched():
            roi_batch_inputs(images, {"det_meta": meta, "bbox_est": xywh}, Ks, ext, depth=depth, depth_factor=factor)

        def per_image():
            nonlocal grid
            if grid is None:
                xs = np.linspace(0, 1, W, endpoint=False, dtype=np.float32)
                ys = np.linspace(0, 1, H, endpoint=False, dtype=np.float32)
                grid = torch.from_numpy(np.ascontiguousarray(np.asarray(np.meshgrid(xs, ys)).transpose(1, 2, 0))).to(dev)
            for j, (_, anns) in enumerate(imgs):
                Ms_in, Ms_out = [], []
                for a in anns:
                    x, y, w, h = a["bbox_est"]
                    c = np.array([x + w / 2, y + h / 2])
                    s = min(max(w, h) * 1.5, max(H, W))
                    Ms_in.append(get_affine_transform(c, (s, s), 0, 256))
                    Ms_out.append(get_affine_transform(c, (s, s), 0, 64))
                if anns:
                    crop_resize_image(images[j], np.stack(Ms_in), 256)
                    crop_resize_float(grid, np.stack(Ms_out), 64)
                    crop_resize_float(grid[..., 0].contiguous(), np.stack(Ms_in), 256, nearest=True)

        def gpu_ms(fn, reps=20):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h0 = time.perf_counter()
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / reps, 1e3 * (time.perf_counter() - h0) / reps

        b_gpu, b_host = gpu_ms(batched)
        p_gpu, p_host = gpu_ms(per_image)
        n_rois = int(meta.shape[0])
    out = {
        "workload": f"test loop, {len(ts.records)} images 640x480, {len(rows)} ROIs, {args.precision}, network pose",
        "images_per_s": round(stats["images"] / wall, 1), "rois_per_s": round(len(rows) / wall, 1),
        "images_per_s_one_image_per_forward": round(res[1][2]["images"] / res[1][1], 1),
        "rois_per_s_one_image_per_forward": round(len(res[1][0]) / res[1][1], 1),
        "batches": stats["batches"],
        "stage_s": {"decode_host_thread_sum": round(stats["decode"], 3), **{k: round(stats[k], 4) for k in
                    ("h2d", "roi_build", "forward", "post", "d2h")}, "csv": round(csv_s, 4), "wall": round(wall, 3)},
        "roi_build_one_batch": {"rois": n_rois, "images": len(imgs), "batched_ms_per_call": round(b_gpu, 4),
                                "batched_host_ms": round(b_host, 3), "per_image_path_ms": round(p_gpu, 4),
                                "per_image_host_ms": round(p_host, 3)},
        "card": name,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
