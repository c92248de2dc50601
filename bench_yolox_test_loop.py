"""Throughput of the YOLOX dataset test loop (yolox_evaluator.yolox_inference_on_dataset) on a synthetic BOP split.

Writes ``--images`` 640 x 480 random BGR PNGs with scene_gt / scene_gt_info / mask_visib (ycbv_bop_test layout) into a
temporary directory, builds seeded YOLOX-X weights (synthetic.make_yolox_state_dict, depth 1.33, width 1.25, 21
classes) and prints one JSON line with the card name and power limit:
  * images/s of the loop at max_batch 1 (the reference's total_batch_size=1) and 8, plain and TTA (the shipped 5
    scales), in bf16x3 and bf16, with the shipped test_size 640 x 640 and conf_thr 0.001: the median, min and max over
    ``--repeats`` timed passes after one warm-up pass that captures the CUDA graphs (kept across passes);
  * the per-stage seconds of the median pass: decode (host, summed over the decoder threads, which overlap the device),
    h2d / letterbox / forward / post / d2h (CUDA events), json (host: box math + the three files);
  * the letterbox kernel against host cv2 (the reference's two preproc passes) for a batch of 8 images of 640 x 480 and
    of 720 x 540;
  * coco_eval.evaluate_boxes against the NumPy COCOeval oracle on the detections of the first 16 images.
With synthetic weights every anchor clears conf_thr 0.001, so the class-aware NMS sees every anchor (DESIGN §7b).
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


def write_masks(root):
    import cv2

    split = os.path.join(root, "BOP_DATASETS", "ycbv", "test")
    for scene in sorted(s for s in os.listdir(split) if s.isdigit()):
        sdir = os.path.join(split, scene)
        info = json.load(open(os.path.join(sdir, "scene_gt_info.json")))
        os.makedirs(os.path.join(sdir, "mask_visib"), exist_ok=True)
        for im_id, insts in info.items():
            for k, g in enumerate(insts):
                m = np.zeros((480, 640), np.uint8)
                x, y, w, h = g["bbox_obj"]
                m[max(y, 0):max(min(y + h, 480), 0), max(x, 0):max(min(x + w, 640), 0)] = 255
                cv2.imwrite(os.path.join(sdir, "mask_visib", f"{int(im_id):06d}_{k:06d}.png"), m)


def host_letterbox(img, test_size):
    """The reference's pre-processing with host cv2: load_resized_img, then ValTransform(legacy=False)."""
    import cv2

    from gdrnpp_bop2022_b200.predictor_yolo import preproc

    r = min(test_size[0] / img.shape[0], test_size[1] / img.shape[1])
    img1 = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR).astype(np.uint8)
    return preproc(img1, test_size)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=48)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from types import SimpleNamespace

    from gdrnpp_bop2022_b200 import yolox_evaluator as YE
    from gdrnpp_bop2022_b200.coco_eval import evaluate_boxes
    from gdrnpp_bop2022_b200.native_ops import yolox_letterbox
    from gdrnpp_bop2022_b200.synthetic import make_yolox_state_dict, write_bop_tree
    from gdrnpp_bop2022_b200.yolox_model import YOLOX
    from oracle import coco_eval_oracle as CO
    from oracle.yolox_oracle import yolox_forward

    dev = torch.device("cuda:0")
    out = {"card": card(), "images": args.images}
    sd = make_yolox_state_dict(yolox_forward, 1.33, 1.25, 21, seed=0, calib_hw=(640, 640), calib_batch=2, device=dev)
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "datasets")
        write_bop_tree(root, num_images=args.images, num_scenes=3, seed=1, with_depth=False)
        write_masks(root)
        ts = YE.YoloxTestSet("ycbv_bop_test", root)
        runs, recs = {}, None
        for precision in ("bf16x3", "bf16"):
            model = YOLOX(1.33, 1.25, 21, max_batch=8, precision=precision).eval()
            model.load_state_dict(sd)
            model.to(dev)
            for augment in (False, True):
                cfg = SimpleNamespace(test_size=(640, 640), conf_thr=0.001, nms_thr=0.65, augment=augment,
                                      scales=(1, 0.75, 0.83, 1.12, 1.25) if augment else None,
                                      test_dataset_names=("ycbv_bop_test",))
                for mb in (1, 8):
                    graphs = {}
                    YE.yolox_inference_on_dataset(cfg, model, root, max_batch=mb, test_set=ts, graph_cache=graphs)
                    passes = []
                    for _ in range(args.repeats):
                        st = {}
                        rec = YE.yolox_inference_on_dataset(cfg, model, root, max_batch=mb, test_set=ts, stats=st,
                                                            graph_cache=graphs)
                        passes.append(st)
                    rates = sorted(p["images"] / p["wall"] for p in passes)
                    st = sorted(passes, key=lambda p: p["images"] / p["wall"])[len(passes) // 2]
                    del graphs
                    t0 = time.perf_counter()
                    YE.YoloxDatasetEvaluator(cfg, SimpleNamespace(obj_ids=ts.obj_ids, gt=None), os.path.join(tmp, "o"),
                                             config_name="bench").evaluate(rec, log=lambda *a: None)
                    st["json"] = time.perf_counter() - t0
                    key = f"{precision}_{'tta' if augment else 'plain'}_b{mb}"
                    runs[key] = {"images_per_s": round(st["images"] / st["wall"], 2),
                                 "images_per_s_range": [round(rates[0], 2), round(rates[-1], 2)],
                                 **{k: round(st[k], 4) for k in ("decode", "h2d", "letterbox", "forward", "post", "d2h",
                                                                 "wall", "json")}}
                    if key == "bf16x3_plain_b8":
                        recs = rec
            del model
            torch.cuda.empty_cache()
        out["loop"] = runs
        # letterbox kernel vs host cv2 (two preproc passes), one batch of 8
        lb = {}
        for H, W in ((480, 640), (540, 720)):
            imgs = np.random.RandomState(0).randint(0, 256, (8, H, W, 3)).astype(np.uint8)
            d = torch.from_numpy(imgs).to(dev)
            x = torch.empty((8, 3, 640, 640), device=dev)
            for _ in range(5):
                yolox_letterbox(d, (640, 640), out=x)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(50):
                yolox_letterbox(d, (640, 640), out=x)
            e1.record()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(5):
                for im in imgs:
                    host_letterbox(im, (640, 640))
            lb[f"{W}x{H}"] = {"kernel_ms": round(e0.elapsed_time(e1) / 50, 4),
                              "host_cv2_ms": round((time.perf_counter() - t0) / 5 * 1e3, 3)}
        out["letterbox_batch8"] = lb
        # coco_eval vs the NumPy oracle on the first 16 images' detections
        coco = []
        for r in recs[:16]:
            coco += YE.image_records(r["image_id"], r["scene_im"], r["dets"], r["hw"], (640, 640), 0.0)[0]
        keep = set(ts.image_ids[:16])
        gt = {"images": [i for i in ts.gt["images"] if i in keep],
              "annotations": [a for a in ts.gt["annotations"] if a["image_id"] in keep]}
        evaluate_boxes(gt, coco, 21, device=dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g = evaluate_boxes(gt, coco, 21, device=dev)
        t_gpu = time.perf_counter() - t0
        t0 = time.perf_counter()
        o = CO.evaluate_boxes(gt, coco, 21)
        t_cpu = time.perf_counter() - t0
        out["coco_eval"] = {"detections": len(coco), "gt": len(gt["annotations"]), "gpu_s": round(t_gpu, 4),
                            "numpy_oracle_s": round(t_cpu, 3),
                            "max_stat_diff": float(np.abs(np.array(g["stats"]) - np.array(o["stats"])).max())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
