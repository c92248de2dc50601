"""CPU oracle of COCO bbox evaluation: a NumPy restatement of pycocotools' COCOeval (iouType "bbox", useCats=1) --
computeIoU / evaluateImg / accumulate / summarize -- written from its documented algorithm.

Inputs are those of gdrnpp_bop2022_b200.coco_eval.evaluate_boxes: gt = {"images": [image_id, ...], "annotations":
[{id, image_id, category_id, bbox (xywh), area, iscrowd}]}, dets = [{image_id, category_id, bbox, score}] (ids 1.. in
list order and area = w * h, as COCO.loadRes assigns them), categories 0 .. num_classes - 1.
"""
import numpy as np

IOU_THRS = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1, endpoint=True)
REC_THRS = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]


def bb_iou(dt, gt, iscrowd):
    """maskApi.c bbIou: [D, G]; no +1, crowd GT divide by the detection area."""
    o = np.zeros((len(dt), len(gt)))
    for g, G in enumerate(gt):
        ga = G[2] * G[3]
        for d, D in enumerate(dt):
            da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            u = da if iscrowd[g] else da + ga - i
            o[d, g] = i / u
    return o


class COCOevalBBox:
    def __init__(self, gt, dets, num_classes):
        self.img_ids = sorted(set(int(i) for i in gt["images"]))
        self.cat_ids = list(range(num_classes))
        self._gts, self._dts = {}, {}
        for k, a in enumerate(gt["annotations"]):
            g = dict(a)
            g.setdefault("id", k + 1)
            g["ignore"] = int(bool(g.get("iscrowd", 0)))
            self._gts.setdefault((int(g["image_id"]), int(g["category_id"])), []).append(g)
        for k, d in enumerate(dets):
            d = dict(d, id=k + 1, iscrowd=0)
            d["area"] = d["bbox"][2] * d["bbox"][3]
            self._dts.setdefault((int(d["image_id"]), int(d["category_id"])), []).append(d)

    def compute_iou(self, img, cat):
        gt, dt = self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in inds][:MAX_DETS[-1]]
        if len(dt) == 0 or len(gt) == 0:
            return []
        return bb_iou([d["bbox"] for d in dt], [g["bbox"] for g in gt], [int(g["iscrowd"]) for g in gt])

    def evaluate_img(self, img, cat, a_rng, max_det):
        gt, dt = self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        if len(gt) == 0 and len(dt) == 0:
            return None
        g_ig = [1 if (g["ignore"] or g["area"] < a_rng[0] or g["area"] > a_rng[1]) else 0 for g in gt]
        gtind = np.argsort(g_ig, kind="mergesort")
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in dtind[0:max_det]]
        iscrowd = [int(o["iscrowd"]) for o in gt]
        ious = self.ious[img, cat]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(IOU_THRS), len(gt), len(dt)
        gtm, dtm = np.zeros((T, G)), np.zeros((T, D))
        gt_ig = np.array([g_ig[i] for i in gtind])
        dt_ig = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gt_ig[m] == 0 and gt_ig[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dt_ig[tind, dind] = gt_ig[m]
                    dtm[tind, dind] = gt[m]["id"]
                    gtm[tind, m] = d["id"]
        a = np.array([d["area"] < a_rng[0] or d["area"] > a_rng[1] for d in dt]).reshape((1, len(dt)))
        dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {"dtIds": [d["id"] for d in dt], "gtIds": [g["id"] for g in gt], "dtMatches": dtm, "gtMatches": gtm,
                "dtScores": [d["score"] for d in dt], "gtIgnore": gt_ig, "dtIgnore": dt_ig}

    def evaluate(self):
        self.ious = {(i, c): self.compute_iou(i, c) for i in self.img_ids for c in self.cat_ids}
        self.eval_imgs = [self.evaluate_img(i, c, a, MAX_DETS[-1]) for c in self.cat_ids for a in AREA_RNG
                          for i in self.img_ids]
        return self

    def accumulate(self):
        T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(self.cat_ids), len(AREA_RNG), len(MAX_DETS)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        I0 = len(self.img_ids)
        for k in range(K):
            for a in range(A):
                for m, max_det in enumerate(MAX_DETS):
                    E = [e for e in self.eval_imgs[k * A * I0 + a * I0:k * A * I0 + (a + 1) * I0] if e is not None]
                    if len(E) == 0:
                        continue
                    dt_scores = np.concatenate([e["dtScores"][0:max_det] for e in E])
                    inds = np.argsort(-dt_scores, kind="mergesort")
                    dtm = np.concatenate([e["dtMatches"][:, 0:max_det] for e in E], axis=1)[:, inds]
                    dt_ig = np.concatenate([e["dtIgnore"][:, 0:max_det] for e in E], axis=1)[:, inds]
                    gt_ig = np.concatenate([e["gtIgnore"] for e in E])
                    npig = np.count_nonzero(gt_ig == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dt_ig))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist()
                        q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        pis = np.searchsorted(rc, REC_THRS, side="left")
                        try:
                            for ri, pi in enumerate(pis):
                                q[ri] = pr[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
        self.precision, self.recall = precision, recall
        return self


def summarize(precision, recall):
    """COCOeval.summarize for bbox: the 12 stats."""
    def one(ap, iou_thr=None, area="all", max_dets=100):
        aind = [i for i, lbl in enumerate(AREA_LBL) if lbl == area]
        mind = [i for i, m in enumerate(MAX_DETS) if m == max_dets]
        if ap == 1:
            s = precision
            if iou_thr is not None:
                s = s[np.where(iou_thr == IOU_THRS)[0]]
            s = s[:, :, :, aind, mind]
        else:
            s = recall
            if iou_thr is not None:
                s = s[np.where(iou_thr == IOU_THRS)[0]]
            s = s[:, :, aind, mind]
        return -1.0 if len(s[s > -1]) == 0 else float(np.mean(s[s > -1]))

    return [one(1), one(1, 0.5, max_dets=100), one(1, 0.75, max_dets=100), one(1, area="small"), one(1, area="medium"),
            one(1, area="large"), one(0, max_dets=1), one(0, max_dets=10), one(0, max_dets=100), one(0, area="small"),
            one(0, area="medium"), one(0, area="large")]


def evaluate_boxes(gt, dets, num_classes):
    """-> {"stats", "precision", "recall", "evaluator"} (the evaluator keeps evalImgs for match-level comparisons)."""
    ev = COCOevalBBox(gt, dets, num_classes).evaluate().accumulate()
    return {"stats": summarize(ev.precision, ev.recall), "precision": ev.precision, "recall": ev.recall, "evaluator": ev}
