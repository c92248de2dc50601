"""The detector's dataset test loop of the reference (test_yolox.sh -> main_yolox.py --eval-only ->
YOLOX_DefaultTrainer.test -> yolox_inference_on_dataset -> YOLOX_COCOEvaluator), with several images in each forward.

  * images: the sorted unique (scene_id, im_id) of <dataset>/test_targets_bop19.json, read as 3-channel BGR (a gray
    image is replicated); where GT is used, an image without instances of the split's objects is dropped, and on
    ycbv_bop_test also an instance whose mask_visib sums to less than 3 (the other splits only count those and keep
    them, with COCO area 0); COCO image ids follow each split's loader (det/yolox/data/datasets/*_bop_test.py);
  * batches: at most ``max_batch`` consecutive images of one size.  A thread pool decodes batch k+1 into pinned staging
    while batch k runs; per batch one H2D copy, the letterbox kernel (native_ops.yolox_letterbox, bit-exact to the
    reference's two cv2 pre-processing passes), the forward (plain or multi-scale TTA; a CUDA graph per batch size),
    yolox_post.postprocess_padded (class-aware, one NMS workspace for the loop) and one D2H copy;
  * outputs: the reference's box math (float32 torch on the CPU: boxes / scale, xyxy -> xywh, obj_conf * cls_conf),
    coco_instances_results.json and coco_instances_results_bop.json as YOLOX_COCOEvaluator writes them, the detection
    file of the pose loop in convert_det_to_our_format.py's save_json layout, and COCO box AP (coco_eval) where the
    split has GT.

Deviations from the reference: the ``time`` of an image is its share of its batch's wall time (batch time / images in
the batch), as in gdrn_evaluator; instances_predictions.pth is not written, since it holds detectron2 objects.
"""
import json
import os
import threading
import time
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import bop_eval
from .gdrn_evaluator import image_shape, pack_batches, read_image
from .native_ops import letterbox_workspace, yolox_letterbox
from .yolox_model import tta_scales
from .yolox_post import postprocess_padded

# DATASETS.TEST name -> Split (det/yolox/data/datasets/*_bop_test.py SPLITS_* and their load()):
#   dataset, image directory under BOP_DATASETS/<dataset>, (colour dir, extension), GT used, obj_id of every label,
#   drop_small_masks: an instance whose mask_visib sums to < 3 is dropped (only ycbv_bop_test's loader skips it; the
#     others count it and keep it),
#   global_image_id: the COCO image_id is a counter over every image of the targets file, dropped ones included
#     (ycbv, hb); otherwise it is the BOP im_id.
Split = namedtuple("Split", "dataset image_dir color has_gt obj_ids drop_small_masks global_image_id")
SPLITS = {
    "ycbv_bop_test": Split("ycbv", "test", ("rgb", ".png"), True, list(range(1, 22)), True, True),
    "lmo_bop_test": Split("lmo", "test", ("rgb", ".png"), True, [1, 5, 6, 8, 9, 10, 11, 12], False, False),
    "tless_bop_test_primesense": Split("tless", "test_primesense", ("rgb", ".png"), True, list(range(1, 31)), False, False),
    "tudl_bop_test": Split("tudl", "test", ("rgb", ".png"), True, [1, 2, 3], False, False),
    "icbin_bop_test": Split("icbin", "test", ("rgb", ".png"), True, [1, 2], False, False),
    "itodd_bop_test": Split("itodd", "test", ("gray", ".tif"), False, list(range(1, 29)), False, False),
    "hb_test_primesense_bop19": Split("hb", "test", ("rgb", ".png"), False, list(range(1, 34)), False, True),
}


def check_test_config(cfg):
    """Reject the settings this loop does not implement, naming the setting (cfg: load_yolox_config's namespace)."""
    if getattr(cfg, "filter_scene", False):
        raise NotImplementedError("YOLOX_COCOEvaluator(filter_scene=True) is not supported")
    if getattr(cfg, "eval_cached", False):
        raise NotImplementedError("val.eval_cached=True (re-evaluating instances_predictions.pth) is not supported")
    if getattr(cfg, "legacy", False):
        raise NotImplementedError("ValTransform(legacy=True) (RGB mean/std normalisation) is not supported")
    names = tuple(getattr(cfg, "test_dataset_names", ()))
    if len(names) != 1:
        raise NotImplementedError(f"test.test_dataset_names={list(names)!r}: the loop runs exactly one test dataset")
    if names[0] not in SPLITS:
        raise NotImplementedError(f"DATASETS.TEST={names[0]!r} is not one of {sorted(SPLITS)}")


def precision_of(cfg, precision=None):
    """half_test or amp_test select bf16 (as YoloPredictor(fp16=True) does), otherwise bf16x3; an explicit one wins."""
    if precision:
        return precision
    return "bf16" if (getattr(cfg, "half_test", False) or getattr(cfg, "amp_test", False)) else "bf16x3"


class YoloxTestSet:
    """Images (and, where the split uses it, COCO GT) of one BOP test split as the reference's *_bop_test.py builds
    them.  .images [(scene_id, im_id)], .image_ids (the COCO image_id of each), .paths, .obj_ids (label -> obj_id),
    .gt (None or {"images": [image_id], "annotations": [...]}).  Where the split's image ids repeat across scenes (BOP
    im_ids of T-LESS), COCO evaluation merges those images, as pycocotools does with the reference's GT."""

    def __init__(self, test_name, datasets_root):
        if test_name not in SPLITS:
            raise NotImplementedError(f"DATASETS.TEST={test_name!r} is not one of {sorted(SPLITS)}")
        self.name = test_name
        sp = SPLITS[test_name]
        self.dataset, self.has_gt, self.obj_ids = sp.dataset, sp.has_gt, sp.obj_ids
        color_dir, ext = sp.color
        self.base = os.path.join(datasets_root, "BOP_DATASETS", self.dataset)
        self.split_dir = os.path.join(self.base, sp.image_dir)
        targets = bop_eval.load_json(os.path.join(self.base, "test_targets_bop19.json"))
        images = sorted({(int(t["scene_id"]), int(t["im_id"])) for t in targets})
        self.images, self.image_ids, self.paths, anns = [], [], [], []
        scene_gt, scene_info = {}, {}
        for n, (scene_id, im_id) in enumerate(images):
            sdir = os.path.join(self.split_dir, f"{scene_id:06d}")
            image_id = n if sp.global_image_id else im_id
            cur = []
            if self.has_gt:
                if scene_id not in scene_gt:
                    scene_gt[scene_id] = bop_eval.load_json(os.path.join(sdir, "scene_gt.json"))
                    scene_info[scene_id] = bop_eval.load_json(os.path.join(sdir, "scene_gt_info.json"))
                for k, g in enumerate(scene_gt[scene_id][str(im_id)]):
                    if int(g["obj_id"]) not in self.obj_ids:
                        continue
                    m = read_mask(os.path.join(sdir, "mask_visib", f"{im_id:06d}_{k:06d}.png"))
                    if sp.drop_small_masks and int(m.sum(dtype=np.int64)) < 3:
                        continue
                    cur.append({"category_id": self.obj_ids.index(int(g["obj_id"])), "iscrowd": 0,
                                "area": int(np.count_nonzero(m)),   # convert_to_coco_json: the area of the mask's RLE
                                "bbox": [float(v) for v in scene_info[scene_id][str(im_id)][k]["bbox_obj"]]})
                if not cur:
                    continue
            self.images.append((scene_id, im_id))
            self.image_ids.append(image_id)
            self.paths.append(os.path.join(sdir, color_dir, f"{im_id:06d}{ext}"))
            anns.extend(dict(a, image_id=image_id) for a in cur)
        self.gt = None
        if self.has_gt:
            self.gt = {"images": list(self.image_ids), "annotations": [dict(a, id=k + 1) for k, a in enumerate(anns)]}


def read_mask(path):
    """A mask_visib PNG as stored (mmcv.imread(path, "unchanged"))."""
    import cv2

    m = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if m is None:
        raise FileNotFoundError(path)
    return m


def box_rows(dets, hw, test_size):
    """The reference's per-image box math (convert_to_coco_format_bop) on a [n, 7] float32 CPU tensor ->
    (bboxes xywh [n,4], labels [n], scores [n]), float32 torch on the CPU."""
    img_h, img_w = hw
    bboxes = dets[:, 0:4].clone()
    scale = min(test_size[0] / float(img_h), test_size[1] / float(img_w))
    bboxes /= scale
    bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 0]
    bboxes[:, 3] = bboxes[:, 3] - bboxes[:, 1]
    return bboxes, dets[:, 6], dets[:, 4] * dets[:, 5]


def image_records(image_id, scene_im, dets, hw, test_size, t_img):
    """-> (coco rows, bop rows) of one image in the reference's key order.  The values are those of the reference's
    per-row ``scores[ind].numpy().item()`` / ``bboxes[ind].numpy().tolist()``, converted for the whole image at once."""
    bboxes, labels, scores = box_rows(dets, hw, test_size)
    coco, bop = [], []
    for box, lab, score in zip(bboxes.tolist(), labels.tolist(), scores.tolist()):
        lab = int(lab)
        coco.append({"image_id": int(image_id), "category_id": lab, "score": score, "bbox": box})
        bop.append({"scene_id": int(scene_im[0]), "image_id": int(scene_im[1]), "category_id": lab + 1, "score": score,
                    "bbox": box, "time": t_img})
    return coco, bop


class _Stage:
    def __init__(self, device):
        self.device = device
        self.host = torch.empty(0, dtype=torch.uint8).pin_memory()
        self.dev = torch.empty(0, dtype=torch.uint8, device=device)
        self.h2d_done = None

    def reserve(self, nb):
        """Allocate up front, on the main thread: the decoder thread must not allocate pinned or device memory while
        the main thread captures a CUDA graph."""
        if self.host.numel() < nb:
            self.host = torch.empty(nb, dtype=torch.uint8).pin_memory()
            self.dev = torch.empty(nb, dtype=torch.uint8, device=self.device)

    def layout(self, N, H, W, C):
        nb = N * H * W * C
        assert self.host.numel() >= nb, "stage not reserved for this batch"
        self.nbytes = nb
        self.h = self.host[:nb].view(N, H, W, C)
        self.d = self.dev[:nb].view(N, H, W, C)


@torch.no_grad()
def yolox_inference_on_dataset(cfg, model, datasets_root, *, max_batch=8, use_cuda_graph=True, stats=None, test_set=None,
                               num_workers=8, device="cuda", graph_cache=None):
    """Run the loop -> records [{"image_id", "scene_im", "hw", "dets" [n,7] float32 CPU, "time"}] in image order.
    cfg: load_yolox_config's namespace (test_size, conf_thr, nms_thr, augment, scales, test_dataset_names); model:
    a YOLOX on ``device``.  stats: a dict that receives the per-stage times in seconds: decode (host, summed over
    threads), h2d / letterbox / forward / post / d2h (device events), wall, and the batch and image counts.
    graph_cache: a dict kept by the caller to reuse the CUDA graphs (and their static inputs) of one model across
    calls; by default each call captures its own."""
    device = torch.device(device)
    ts = test_set or YoloxTestSet(cfg.test_dataset_names[0], datasets_root)
    if model.num_classes != len(ts.obj_ids):
        raise ValueError(f"model.head.num_classes={model.num_classes} but {ts.name!r} has {len(ts.obj_ids)} objects")
    if not ts.images:
        return []
    th, tw = (int(v) for v in cfg.test_size)
    augment = bool(getattr(cfg, "augment", False))
    if augment and tta_scales(cfg) is None:
        raise NotImplementedError("test.augment=True needs test.scales")
    keys = [image_shape(p) for p in ts.paths]
    batches = pack_batches([1] * len(keys), max_batch, keys)
    stages = [_Stage(device), _Stage(device)]
    need = max(len(b) * int(np.prod(keys[b[0]])) for b in batches)
    for st in stages:
        st.reserve(need)
    cache = {} if graph_cache is None else graph_cache
    if cache.setdefault("model", model) is not model:
        raise ValueError("graph_cache holds the graphs of another model")
    scales = tta_scales(cfg) if augment else None
    stream = torch.cuda.current_stream(device)
    timing = stats is not None
    ev = lambda: torch.cuda.Event(enable_timing=True)
    dec_time = [0.0]
    lock = threading.Lock()
    lb_ws, post_ws = {}, [None]

    def fill(stage, batch):
        H, W, C = keys[batch[0]]
        stage.layout(len(batch), H, W, C)

        def one(j):
            t0 = time.perf_counter()
            im = read_image(ts.paths[batch[j]])
            if im.shape != (H, W, C):
                raise ValueError(f"{ts.paths[batch[j]]}: {im.shape} in a batch of {(H, W, C)} images")
            stage.h[j].numpy()[...] = im
            with lock:
                dec_time[0] += time.perf_counter() - t0

        list(pool.map(one, range(len(batch))))
        return batch

    def static_input(B):
        """The letterbox output of a batch of B: the static input of that batch size's graph."""
        key = ("input", B, th, tw, scales)
        if key not in cache:
            cache[key] = torch.empty((B, 3, th, tw), dtype=torch.float32, device=device)
        return cache[key]

    def forward(x):
        B = x.shape[0]
        kw = {"augment": True, "cfg": cfg} if augment else {}
        if not use_cuda_graph or B > model.max_batch:
            return model(x, **kw)["det_preds"]
        key = ("graph", B, th, tw, scales)
        if key not in cache:
            cache[key] = model.capture_graph(x, augment=augment, cfg=cfg if augment else None)
        replay, out = cache[key]
        replay()
        return out["det_preds"]

    records = []
    pending = None
    tstat = {"h2d": [], "letterbox": [], "forward": [], "post": [], "d2h": []}
    pool = ThreadPoolExecutor(num_workers)
    feeder = ThreadPoolExecutor(1)
    t_start = time.perf_counter()
    t_last = [t_start]

    def finish(p):
        batch, host_dets, host_n, done = p
        done.synchronize()
        now = time.perf_counter()
        share = (now - t_last[0]) / len(batch)
        t_last[0] = now
        counts = host_n.tolist()
        for j, idx in enumerate(batch):
            records.append({"image_id": ts.image_ids[idx], "scene_im": ts.images[idx], "hw": keys[idx][:2],
                            "dets": host_dets[j, :counts[j]].clone(), "time": share})

    try:
        with torch.cuda.device(device):
            fut = feeder.submit(fill, stages[0], batches[0])
            for bi in range(len(batches)):
                stage = stages[bi % 2]
                batch = fut.result()
                if bi + 1 < len(batches):
                    nxt = stages[(bi + 1) % 2]
                    if nxt.h2d_done is not None:
                        nxt.h2d_done.synchronize()
                    fut = feeder.submit(fill, nxt, batches[bi + 1])
                e = [ev() for _ in range(6)] if timing else None
                if timing:
                    e[0].record(stream)
                stage.dev[:stage.nbytes].copy_(stage.host[:stage.nbytes], non_blocking=True)
                stage.h2d_done = torch.cuda.Event()
                stage.h2d_done.record(stream)
                if timing:
                    e[1].record(stream)
                B, H, W, C = stage.d.shape
                x = static_input(B)
                if (B, H, W) not in lb_ws:
                    lb_ws[(B, H, W)] = letterbox_workspace(B, H, W, (th, tw), device)
                yolox_letterbox(stage.d, (th, tw), out=x, workspace=lb_ws[(B, H, W)])
                if timing:
                    e[2].record(stream)
                det_preds = forward(x)
                if timing:
                    e[3].record(stream)
                dets, n_det = postprocess_padded(det_preds, model.num_classes, cfg.conf_thr, cfg.nms_thr,
                                                 workspace=post_ws)
                if timing:
                    e[4].record(stream)
                host_dets = torch.empty(dets.shape, dtype=torch.float32, pin_memory=True)
                host_n = torch.empty(n_det.shape, dtype=torch.int32, pin_memory=True)
                host_dets.copy_(dets, non_blocking=True)
                host_n.copy_(n_det, non_blocking=True)
                done = torch.cuda.Event()
                done.record(stream)
                if timing:
                    e[5].record(stream)
                    for k, (a, b) in zip(("h2d", "letterbox", "forward", "post", "d2h"), zip(e[:-1], e[1:])):
                        tstat[k].append((a, b))
                if pending is not None:
                    finish(pending)
                pending = (batch, host_dets, host_n, done)
            if pending is not None:
                finish(pending)
    finally:
        pool.shutdown()
        feeder.shutdown()
    if timing:
        torch.cuda.synchronize(device)
        stats.update({k: sum(a.elapsed_time(b) for a, b in v) / 1e3 for k, v in tstat.items()})
        stats["decode"] = dec_time[0]
        stats["wall"] = time.perf_counter() - t_start
        stats["batches"] = len(batches)
        stats["images"] = len(records)
    return records


def save_json(path, content):
    """convert_det_to_our_format.py's save_json (sort=False) for a dict: one key per line, values sort_keys."""
    with open(path, "w") as f:
        f.write("{\n")
        for i, (k, v) in enumerate(content.items()):
            f.write('  "{}": {}'.format(k, json.dumps(v, sort_keys=True)))
            if i != len(content) - 1:
                f.write(",")
            f.write("\n")
        f.write("}")


def convert_det_to_ours(bop_rows, obj_ids):
    """convert_det_to_our_format.py / convert_lmo_det_to_ours.py: {"scene/im": [{bbox_est, obj_id, score, time}]},
    obj_id = obj_ids[category_id - 1] (category_id = label + 1)."""
    outs = {}
    for d in bop_rows:
        outs.setdefault(f"{d['scene_id']}/{d['image_id']}", []).append(
            {"bbox_est": d["bbox"], "obj_id": obj_ids[d["category_id"] - 1], "score": d["score"], "time": d["time"]})
    return outs


class YoloxDatasetEvaluator:
    """Writes the reference's result files for the loop's records and scores COCO box AP where the split has GT."""

    def __init__(self, cfg, test_set, output_dir, det_file=None, config_name="yolox"):
        self.cfg, self.ts, self.output_dir = cfg, test_set, output_dir
        self.det_file = det_file or os.path.join(output_dir, "test_bboxes", config_name + ".json")

    def evaluate(self, records, log=print):
        ts = self.ts
        coco, bop = [], []
        for r in records:
            c, b = image_records(r["image_id"], r["scene_im"], r["dets"], r["hw"], self.cfg.test_size, r["time"])
            coco += c
            bop += b
        os.makedirs(self.output_dir, exist_ok=True)
        files = {"coco": os.path.join(self.output_dir, "coco_instances_results.json"),
                 "bop": os.path.join(self.output_dir, "coco_instances_results_bop.json"), "det_file": self.det_file}
        for key, content in (("coco", coco), ("bop", bop)):
            with open(files[key], "w") as f:
                f.write(json.dumps(content))
        os.makedirs(os.path.dirname(os.path.abspath(self.det_file)), exist_ok=True)
        save_json(self.det_file, convert_det_to_ours(bop, ts.obj_ids))
        log("instances_predictions.pth is not written (it holds detectron2 objects)")
        res = {"files": files}
        if ts.gt is None:
            log("Annotations are not available for evaluation.")
            return res
        from .coco_eval import METRICS, evaluate_boxes

        ap = evaluate_boxes(ts.gt, coco, len(ts.obj_ids), obj_ids=ts.obj_ids)
        res["bbox"] = {k: v for k, v in ap.items() if k in METRICS or k.startswith(("AP-", "AR-"))}
        log("Evaluation results for bbox: " + json.dumps({k: round(ap[k], 3) for k in METRICS}))
        return res
