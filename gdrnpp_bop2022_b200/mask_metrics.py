"""The reference's mask tools (core/gdrn_modeling/tools/compute_mIoU_mask.py and compute_f1_score_mask.py) on a
results.pkl of the save-results loop, for a BOP test split:

    python -m gdrnpp_bop2022_b200.mask_metrics --dataset lmo_bop_test --obj_id 1 --res_path .../results.pkl \\
        [--mask_type vis|full] [--height 480 --width 640] --datasets_root datasets

For every image of the split (the sorted unique (scene_id, im_id) of test_targets_bop19.json): the first prediction of
the object is decoded at --height x --width and compared with the first GT instance of the object in scene_gt.json
(mask_visib/{im:06d}_{k:06d}.png for ``vis``, mask/... for ``full``, read as astype(bool)); an image missing from the
results, or without a prediction of the object, scores 0.  mIoU is compute_mean_iou (the mean of I / U over the labels
present in the GT), F1 is sklearn's binary f1_score (2 TP / (2 TP + FP + FN), 0 when that is 0 / 0).  Both come from
one batched GPU decode + confusion count over all compared images (native_ops.rle_confusion); the GT PNGs are decoded
on a thread pool.

Deviations from the reference: ``--obj_id`` replaces ``--cls`` (this package has no object names) and the LM-only
name assertions are dropped; an image whose GT has no instance of the object is skipped and counted (the reference
reuses the previous image's GT mask there, or fails on the first image).
"""
import argparse
import os
import pickle
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import bop_eval
from .gdrn_evaluator import image_list


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="mIoU and F1 of the saved masks of one object")
    ap.add_argument("--dataset", required=True, help="DATASETS.TEST name, e.g. lmo_bop_test")
    ap.add_argument("--obj_id", type=int, required=True)
    ap.add_argument("--mask_type", default="vis", help="vis | full")
    ap.add_argument("--res_path", required=True, help="results.pkl of the save-results loop")
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--datasets_root", default="datasets")
    ap.add_argument("--num_workers", type=int, default=8)
    return ap.parse_args(argv)


def metrics_from_counts(counts):
    """[P,4] TP, FP, FN, TN -> (mIoU [P], F1 [P]) as compute_mean_iou and binary f1_score compute them."""
    c = np.asarray(counts, np.float64).reshape(-1, 4)
    tp, fp, fn, tn = c.T
    has1, has0 = tp + fn > 0, fp + tn > 0   # labels present in the GT
    iou1 = np.divide(tp, tp + fp + fn, out=np.zeros_like(tp), where=has1)
    iou0 = np.divide(tn, tn + fp + fn, out=np.zeros_like(tn), where=has0)
    miou = (iou1 * has1 + iou0 * has0) / np.maximum(has1.astype(np.float64) + has0, 1)
    d = 2 * tp + fp + fn
    f1 = np.divide(2 * tp, d, out=np.zeros_like(tp), where=d > 0)
    return miou, f1


def _read_gt(path, H, W):
    import cv2

    m = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if m is None:
        raise FileNotFoundError(path)
    if m.shape[:2] != (H, W):
        raise ValueError(f"{path}: {m.shape[:2]} GT mask, --height/--width give {(H, W)}")
    return m.reshape(H, W, -1)[..., 0].astype(bool)


def run(args):
    from . import yolox_evaluator
    from .native_ops import rle_confusion

    if args.mask_type not in ("vis", "full"):
        raise ValueError(f"Unknown mask type: {args.mask_type}, available options: vis | full")
    if args.dataset not in yolox_evaluator.SPLITS:
        raise ValueError(f"--dataset {args.dataset!r} is not one of {sorted(yolox_evaluator.SPLITS)}")
    split = yolox_evaluator.SPLITS[args.dataset]
    if not split.has_gt:
        raise ValueError(f"{args.dataset} has no GT masks")
    print("evaluating visible mask" if args.mask_type == "vis" else "evaluating full mask")
    print("dataset: ", args.dataset)
    print("object id: ", args.obj_id)
    print("results path: ", args.res_path)
    base = os.path.join(args.datasets_root, "BOP_DATASETS", split.dataset)
    images = image_list(bop_eval.load_json(os.path.join(base, "test_targets_bop19.json")))
    with open(args.res_path, "rb") as f:
        res = pickle.load(f)
    key = "mask" if args.mask_type == "vis" else "full_mask"
    mask_dir = "mask_visib" if args.mask_type == "vis" else "mask"
    H, W = args.height, args.width
    slots, rles, paths = [], [], []   # slots: None = scored 0, else the index of the compared pair
    num_detected = skipped = 0
    scene_gt = {}
    for scene_id, im_id in images:
        preds = res.get(f"{scene_id}/{im_id}")
        pred_ids = [int(p["obj_id"]) for p in preds] if preds is not None else []
        if args.obj_id not in pred_ids:
            slots.append(None)
            continue
        sdir = os.path.join(base, split.image_dir, f"{scene_id:06d}")
        if scene_id not in scene_gt:
            scene_gt[scene_id] = bop_eval.load_json(os.path.join(sdir, "scene_gt.json"))
        gts = [int(g["obj_id"]) for g in scene_gt[scene_id][str(im_id)]]
        if args.obj_id not in gts:
            skipped += 1
            continue
        num_detected += 1
        slots.append(len(rles))
        rles.append(preds[pred_ids.index(args.obj_id)][key])
        paths.append(os.path.join(sdir, mask_dir, f"{im_id:06d}_{gts.index(args.obj_id):06d}.png"))
    gt = np.zeros((len(paths), H, W), np.uint8)

    def load(i):
        gt[i] = _read_gt(paths[i], H, W)

    with ThreadPoolExecutor(args.num_workers) as pool:
        list(pool.map(load, range(len(paths))))
    rles = [dict(r, size=[H, W]) for r in rles]   # cocosegm2mask decodes the string at --height x --width
    miou_c, f1_c = metrics_from_counts(rle_confusion(rles, gt)) if rles else (np.zeros(0), np.zeros(0))
    mious = np.array([0.0 if s is None else miou_c[s] for s in slots])
    f1s = np.array([0.0 if s is None else f1_c[s] for s in slots])
    miou, f1 = float(np.mean(mious)) if len(mious) else float("nan"), float(np.mean(f1s)) if len(f1s) else float("nan")
    print("mask type: {}".format(args.mask_type))
    print("dataset name: ", args.dataset, "object id: ", args.obj_id)
    print("dataset length: ", len(images))
    print("length of mIoUs: ", len(mious))
    print("length of F1 scores: ", len(f1s))
    print("num detected: ", num_detected)
    print("skipped (no GT instance of the object): ", skipped)
    print(f"mIoU (%): {miou * 100:.2f}")
    print(f"mean F1 score (%): {f1 * 100:.2f}")
    return {"miou": miou, "f1": f1, "num_scores": len(mious), "num_detected": num_detected, "skipped": skipped,
            "images": len(images)}


def main(argv=None):
    return run(parse_args(argv))


if __name__ == "__main__":
    main(sys.argv[1:])
