"""COCO box AP on the GPU: pycocotools COCOeval (iouType "bbox") as the reference's YOLOX_COCOEvaluator runs it
(det/yolox/evaluators/yolox_coco_evaluator.py _evaluate_predictions_on_coco + _derive_coco_results), with the matching
of every (image, category) pair and the per-category accumulation in csrc/coco_eval.cu.  The host groups the inputs
into pairs (NumPy, no per-category loop) and computes the 12 summary stats from the precision / recall arrays.

Deviation from the reference: per-category keys are ``AP-obj_XXXXXX`` / ``AR-obj_XXXXXX`` (the obj_id of the label),
since the object names live in the reference's dataset metadata, which this package does not carry.
"""
import numpy as np
import torch

from . import _lib

IOU_THRS = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1, endpoint=True)
REC_THRS = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1, endpoint=True)
MAX_DETS = (1, 10, 100)
AREA_RNG = ((0 ** 2, 1e5 ** 2), (0 ** 2, 32 ** 2), (32 ** 2, 96 ** 2), (96 ** 2, 1e5 ** 2))
AREA_LBL = ("all", "small", "medium", "large")
METRICS = ("AP", "AP50", "AP75", "APs", "APm", "APl")


def summarize(precision, recall):
    """COCOeval.summarize for bbox -> the 12 stats (AP, AP50, AP75, APs/m/l at 100 dets, AR@1/10/100, ARs/m/l)."""
    def one(ap, iou_thr=None, area="all", max_dets=100):
        aind = [i for i, lbl in enumerate(AREA_LBL) if lbl == area]
        mind = [i for i, m in enumerate(MAX_DETS) if m == max_dets]
        s = precision if ap else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap else s[:, :, aind, mind]
        return -1.0 if len(s[s > -1]) == 0 else float(np.mean(s[s > -1]))

    return [one(1), one(1, 0.5), one(1, 0.75), one(1, area="small"), one(1, area="medium"), one(1, area="large"),
            one(0, max_dets=1), one(0, max_dets=10), one(0), one(0, area="small"), one(0, area="medium"),
            one(0, area="large")]


def _group(keys):
    order = np.argsort(keys, kind="stable")
    return order, keys[order]


def evaluate_boxes(gt, dets, num_classes, obj_ids=None, device="cuda", return_matches=False):
    """gt = {"images": [image_id, ...], "annotations": [{image_id, category_id (label), bbox xywh, area, iscrowd,
    optional id}]} (ids default to 1.. in list order), dets = [{image_id, category_id, bbox xywh, score}] on GT images
    (ids 1.. and area w * h, as COCO.loadRes sets them); categories 0 .. num_classes - 1; obj_ids: the obj_id of each
    label for the per-category keys (default label + 1).
    -> {"stats": [12], "precision": [T,R,K,A,M], "recall": [T,K,A,M], "AP", "AP50", "AP75", "APs", "APm", "APl" (x100,
    NaN for a stat of -1 or without detections), "AP-obj_XXXXXX" / "AR-obj_XXXXXX" (x100, NaN without GT)}.
    return_matches adds "matches": the per-pair match arrays, with COCO ids, for comparisons with pycocotools."""
    device = torch.device(device)
    K = int(num_classes)
    obj_ids = list(obj_ids) if obj_ids is not None else list(range(1, K + 1))
    img_ids = np.array(sorted(set(int(i) for i in gt["images"])), np.int64)
    I = len(img_ids)
    anns = gt["annotations"]
    g_img = np.array([int(a["image_id"]) for a in anns], np.int64)
    g_cat = np.array([int(a["category_id"]) for a in anns], np.int64)
    g_box = np.array([a["bbox"] for a in anns], np.float64).reshape(-1, 4)
    g_area = np.array([a["area"] for a in anns], np.float64)
    g_crowd = np.array([int(bool(a.get("iscrowd", 0))) for a in anns], np.uint8)
    g_id = np.array([int(a.get("id", k + 1)) for k, a in enumerate(anns)], np.int64)
    d_img = np.array([int(d["image_id"]) for d in dets], np.int64)
    d_cat = np.array([int(d["category_id"]) for d in dets], np.int64)
    d_box = np.array([d["bbox"] for d in dets], np.float64).reshape(-1, 4)
    d_score = np.array([d["score"] for d in dets], np.float64)
    for name, c in (("annotation", g_cat), ("detection", d_cat)):
        if len(c) and (c.min() < 0 or c.max() >= K):
            raise ValueError(f"a {name} has a category_id outside 0..{K - 1}")
    g_pos, d_pos = np.searchsorted(img_ids, g_img), np.searchsorted(img_ids, d_img)
    for name, pos, ids in (("annotation", g_pos, g_img), ("detection", d_pos, d_img)):
        if len(ids) and (pos.max() >= I or not np.array_equal(img_ids[np.minimum(pos, I - 1)], ids)):
            raise ValueError(f"a {name} is on an image that is not in gt['images']")
    g_perm, g_key = _group(g_cat * I + g_pos)
    d_perm, d_key = _group(d_cat * I + d_pos)
    pair_key = np.union1d(g_key, d_key).astype(np.int64)
    P = len(pair_key)
    pair_gt_off = np.searchsorted(g_key, np.append(pair_key, K * I)).astype(np.int32)
    pair_dt_off = np.searchsorted(d_key, np.append(pair_key, K * I)).astype(np.int32)
    G_p, D_p = np.diff(pair_gt_off), np.diff(pair_dt_off)
    kept = np.minimum(D_p, MAX_DETS[-1])
    pair_kept_off = np.concatenate([[0], np.cumsum(kept)]).astype(np.int32)
    pair_iou_off = np.concatenate([[0], np.cumsum(kept.astype(np.int64) * G_p)]).astype(np.int64)
    first = np.searchsorted(pair_key // max(I, 1), np.arange(K + 1))
    cat_off = pair_kept_off[first].astype(np.int32)
    cat_gt_off = pair_gt_off[first].astype(np.int32)
    cat_pairs = np.diff(first).astype(np.int32)
    Gtot, Dkept = int(pair_gt_off[-1]), int(pair_kept_off[-1])
    T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(MAX_DETS)

    dv = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    e = lambda n, dt: torch.empty((max(int(n), 1),), dtype=dt, device=device)
    with torch.cuda.device(device):
        t_gbox, t_garea, t_gcrowd = dv(g_box[g_perm]), dv(g_area[g_perm]), dv(g_crowd[g_perm])
        t_dbox, t_dscore = dv(d_box[d_perm]), dv(d_score[d_perm])
        t_pg, t_pd, t_pk, t_pi = dv(pair_gt_off), dv(pair_dt_off), dv(pair_kept_off), dv(pair_iou_off)
        t_iou_thrs, t_area = dv(IOU_THRS), dv(np.array(AREA_RNG, np.float64))
        dt_order, kept_score, kept_rank = e(Dkept, torch.int32), e(Dkept, torch.float64), e(Dkept, torch.int32)
        ious = e(pair_iou_off[-1], torch.float64)
        gt_ignore, gt_match = e(A * Gtot, torch.uint8), e(A * T * Gtot, torch.int32)
        dt_match, dt_ignore = e(A * T * Dkept, torch.int32), e(A * T * Dkept, torch.uint8)
        p = _lib.ptr
        L = _lib.lib()
        _lib.check(L.coco_eval_match(p(t_gbox), p(t_garea), p(t_gcrowd), p(t_dbox), p(t_dscore), p(t_pg), p(t_pd), p(t_pk),
                                     p(t_pi), P, Gtot, Dkept, p(t_iou_thrs), T, p(t_area), A, MAX_DETS[-1], p(dt_order),
                                     p(kept_score), p(kept_rank), p(ious), p(gt_ignore), p(dt_match), p(dt_ignore),
                                     p(gt_match), _lib.current_stream()), "coco_eval_match")
        precision = torch.full((T, R, K, A, M), -1.0, dtype=torch.float64, device=device)
        recall = torch.full((T, K, A, M), -1.0, dtype=torch.float64, device=device)
        ws = torch.empty(L.coco_eval_accumulate_workspace_bytes(Dkept), dtype=torch.uint8, device=device)
        # named: a temporary's block would return to the caching allocator before the launch and be reused
        t_co, t_cgo, t_cp = dv(cat_off), dv(cat_gt_off), dv(cat_pairs)
        t_rec, t_md = dv(REC_THRS), dv(np.array(MAX_DETS, np.int32))
        _lib.check(L.coco_eval_accumulate(p(kept_score), p(kept_rank), p(dt_match), p(dt_ignore), p(gt_ignore), p(t_co),
                                          p(t_cgo), p(t_cp), int(np.diff(cat_off).max(initial=0)), K, Dkept, Gtot, T, A,
                                          p(t_rec), R, p(t_md), M, p(ws), ws.numel(), p(precision), p(recall),
                                          _lib.current_stream()),
                   "coco_eval_accumulate")
        precision, recall = precision.cpu().numpy(), recall.cpu().numpy()
    stats = summarize(precision, recall)
    res = {"stats": stats, "precision": precision, "recall": recall}
    has_dets = len(dets) > 0
    res.update({m: float(s * 100) if (has_dets and s >= 0) else float("nan") for m, s in zip(METRICS, stats)})
    for k in range(K):
        pk = precision[:, :, k, 0, -1]
        pk = pk[pk > -1]
        rk = recall[:, k, 0, -1]
        rk = rk[rk > -1]
        res["AP-obj_{:06d}".format(obj_ids[k])] = float(np.mean(pk) * 100) if pk.size else float("nan")
        res["AR-obj_{:06d}".format(obj_ids[k])] = float(np.mean(rk) * 100) if rk.size else float("nan")
    if return_matches:
        det_id = (d_perm + 1).astype(np.int64)                       # loadRes ids, in grouped order
        order = dt_order.cpu().numpy()[:Dkept]
        kept_det_id = det_id[order] if Dkept else np.zeros(0, np.int64)
        gm = gt_match.cpu().numpy()[:A * T * Gtot].reshape(A, T, Gtot)
        dm = dt_match.cpu().numpy()[:A * T * Dkept].reshape(A, T, Dkept)
        grouped_gt_id = g_id[g_perm]
        res["matches"] = {
            "pairs": [(int(img_ids[k % I]), int(k // I)) for k in pair_key], "pair_gt_off": pair_gt_off,
            "pair_kept_off": pair_kept_off, "gt_id": grouped_gt_id, "kept_det_id": kept_det_id,
            "gt_ignore": gt_ignore.cpu().numpy()[:A * Gtot].reshape(A, Gtot),
            "dt_match": np.where(dm > 0, grouped_gt_id[np.maximum(dm - 1, 0)] if Gtot else 0, 0),
            "dt_ignore": dt_ignore.cpu().numpy()[:A * T * Dkept].reshape(A, T, Dkept),
            "gt_match": np.where(gm > 0, kept_det_id[np.maximum(gm - 1, 0)] if Dkept else 0, 0)}
    return res
