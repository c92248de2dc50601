"""YOLOX training batches built on the GPU: what build_yolox_train_loader yields per batch for the shipped detector
configs (configs/yolox/bop_pbr/yolox_x_640_augCozyAAEhsv_*): MosaicDetection.__getitem__
(det/yolox/data/datasets/mosaicdetection.py) over Base_DatasetFromList.pull_item, with its TrainTransform
(det/yolox/data/data_augment.py), for every sample of a batch, collated as torch's default_collate does.

Every random choice is drawn on the host, from one numpy Generator per batch, into a fixed-layout record per sample
(``Sampler.draw``); the box arithmetic follows the reference in float64 on the host.  The device work
(csrc/yolox_train_aug.cu) is a deterministic function of (decoded images, records): the resizes of load_resized_img and
the mosaic tiles, the mosaic seen through the random affine, mixup, TrainTransform's HSV pass, mirror and letterbox,
the wrapper's HSV pass and colour program on the (w, h, c) transpose of the image, and the float32 CHW pack.  Nothing
synchronises within a batch.
"""
import json
import math
import os
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib
from .train_batch import COLOR_OPS, N_FPAR, N_IPAR, _draw_op, dropout_grid, parse_color_aug, read_bgr
from .yolox_evaluator import SPLITS as TEST_SPLITS

GdrnError = _lib.GdrnError

MAX_LABELS = 120   # the wrapper's TrainTransform(max_labels=120) serves both branches; the dataset's own (50) never runs
BORDER = 114

# DATASETS.TRAIN name -> its registrar's constants (det/yolox/data/datasets/*_pbr.py, tless_primesense_train.py,
# tudl_train_real.py): dataset, split directory, image extension, the registrar's (height, width), its visible-area
# rule and filter_invalid (bbox_visib wider and taller than one pixel).  The area rule drops an instance when
# ``area < 30`` (min_area 30) or ``area <= 64`` (min_area 65), where ``area`` is the sum of the mask_visib PNG: its pixel
# count where the registrar casts the mask to bool first (LM / LM-O, ITODD and TUD-L PBR: mask_value 1), 255 times it
# where it sums the raw 0 / 255 PNG (mask_value 255), so that there only an empty mask is dropped.
TrainSplit = namedtuple("TrainSplit", "dataset split ext hw min_area mask_value filter_invalid")
TRAIN_SPLITS = {
    "lmo_pbr_train": TrainSplit("lmo", "train_pbr", ".jpg", (480, 640), 30, 1, True),
    "tless_pbr_train": TrainSplit("tless", "train_pbr", ".jpg", (540, 720), 30, 255, False),
    "tudl_pbr_train": TrainSplit("tudl", "train_pbr", ".jpg", (480, 640), 30, 1, True),
    "icbin_pbr_train": TrainSplit("icbin", "train_pbr", ".jpg", (480, 640), 30, 255, False),
    "itodd_pbr_train": TrainSplit("itodd", "train_pbr", ".jpg", (960, 1280), 30, 1, True),
    "hb_pbr_train": TrainSplit("hb", "train_pbr", ".jpg", (480, 640), 65, 255, True),
    "ycbv_train_pbr": TrainSplit("ycbv", "train_pbr", ".jpg", (480, 640), 65, 255, True),
    "tless_primesense_train": TrainSplit("tless", "train_primesense", ".png", (400, 400), 65, 255, True),
    "tudl_train_real": TrainSplit("tudl", "train_real", ".png", (480, 640), 30, 255, True),
}
# splits whose registrar needs more than scene_gt / scene_gt_info: the reason, for the rejection
UNSUPPORTED_SPLITS = {
    "ycbv_train_real": "its registrar (ycbv_d2.py) lists the images of an image-set file and re-poses some scenes "
                       "for another camera; only the BOP scene-directory registrars are supported",
}
# the test split whose object order gives the labels of each dataset
LABEL_SPLIT = {"lmo": "lmo_bop_test", "ycbv": "ycbv_bop_test", "tless": "tless_bop_test_primesense",
               "tudl": "tudl_bop_test", "icbin": "icbin_bop_test", "itodd": "itodd_bop_test",
               "hb": "hb_test_primesense_bop19"}


def letterbox_size(h, w, th, tw):
    """preproc / load_resized_img's resized size: r = min(th / h, tw / w) -> (int(h r), int(w r)), r."""
    r = min(th / h, tw / w)
    return int(h * r), int(w * r), r


# --------------------------------------------------------------------------------------------- configuration
def check_train_config(cfg):
    """Reject, naming the setting, what the batcher does not build (cfg: load_yolox_config's namespace)."""
    w = cfg.aug_wrapper
    if tuple(cfg.train_img_size) != (640, 640):
        raise NotImplementedError(f"dataloader.train.dataset.img_size={tuple(cfg.train_img_size)}: only the shipped "
                                  "(640, 640) is supported")
    for k in ("mosaic_prob", "mixup_prob"):
        if not 0.0 <= float(w[k]) <= 1.0:
            raise NotImplementedError(f"dataloader.train.aug_wrapper.{k}={w[k]!r} is outside [0, 1]")
    if float(w["COLOR_AUG_PROB"]) > 0:
        if str(w["COLOR_AUG_TYPE"]).lower() != "code":
            raise NotImplementedError(f"dataloader.train.aug_wrapper.COLOR_AUG_TYPE={w['COLOR_AUG_TYPE']!r}: only 'code' "
                                      "(an imgaug program) is supported")
        parse_color_aug(str(w["COLOR_AUG_CODE"]))
    if str(w["FORMAT"]) not in ("RGB", "BGR"):
        raise NotImplementedError(f"dataloader.train.aug_wrapper.FORMAT={w['FORMAT']!r}: only RGB and BGR are supported")
    for k in ("degrees", "translate", "shear", "mosaic_scale", "mixup_scale"):
        v = w[k]
        if not (isinstance(v, (int, float)) or (isinstance(v, (tuple, list)) and len(v) == 2)):
            raise NotImplementedError(f"dataloader.train.aug_wrapper.{k}={v!r}: a number or a (low, high) pair")
    names = list(cfg.train_dataset_names)
    if not names:
        raise GdrnError("DATASETS.TRAIN is empty")
    for n in names:
        if n in UNSUPPORTED_SPLITS:
            raise NotImplementedError(f"DATASETS.TRAIN entry {n!r} is not supported: {UNSUPPORTED_SPLITS[n]}")
        if n not in TRAIN_SPLITS:
            raise NotImplementedError(f"DATASETS.TRAIN entry {n!r} is not one of {sorted(TRAIN_SPLITS)}")


def _aug_param(rng, value, center=0.0):
    """get_aug_params: a number v draws uniform(center - v, center + v), a pair (lo, hi) uniform(lo, hi)."""
    if isinstance(value, (tuple, list)):
        return float(rng.uniform(value[0], value[1]))
    return float(rng.uniform(center - value, center + value))


def affine_matrix(angle, scale, shear_x_deg, shear_y_deg, tx, ty, size):
    """get_affine_matrix from its drawn values: cv2.getRotationMatrix2D about (0, 0), the two shears, the translation
    fractions times the target (w, h)."""
    import cv2

    R = cv2.getRotationMatrix2D(angle=angle, center=(0, 0), scale=scale)
    M = np.ones([2, 3])
    shear_x, shear_y = math.tan(shear_x_deg * math.pi / 180), math.tan(shear_y_deg * math.pi / 180)
    M[0] = R[0] + shear_y * R[1]
    M[1] = R[1] + shear_x * R[0]
    M[0, 2] = tx * size[0]
    M[1, 2] = ty * size[1]
    return M


def hsv_luts(gains):
    """augment_hsv's three LUTs for r = gains: ((x r0) % 180, clip(x r1), clip(x r2)), truncated to uint8."""
    x = np.arange(0, 256, dtype=np.int16)
    return np.stack([((x * gains[0]) % 180).astype(np.uint8), np.clip(x * gains[1], 0, 255).astype(np.uint8),
                     np.clip(x * gains[2], 0, 255).astype(np.uint8)])


# --------------------------------------------------------------------------------------------- the training split
def _load_json(path):
    with open(path) as f:
        return json.load(f)


class YoloxTrainSet:
    """One sample per image of the DATASETS.TRAIN splits, with the registrars' filters (objects of the dataset's test
    split, filter_invalid on bbox_visib, each registrar's visible-area rule (TRAIN_SPLITS) on scene_gt_info's
    px_count_visib, so no mask PNG is decoded; images without instances dropped) and then Base_DatasetFromList.load_anno: bbox_obj XYWH -> XYXY clipped to the
    registrar's image size, area > 0, scaled by r = min(640 / H, 640 / W).  .images[i] = {path, hw, labels [k,5]
    (x1, y1, x2, y2, 0-based class), image_id, scene_im_id}; .obj_ids (label -> obj_id)."""

    def __init__(self, cfg, datasets_root):
        check_train_config(cfg)
        names = list(cfg.train_dataset_names)
        dss = {TRAIN_SPLITS[n].dataset for n in names}
        if len(dss) != 1:
            raise GdrnError(f"DATASETS.TRAIN mixes datasets {sorted(dss)}; one dataset per batcher")
        self.dataset = dss.pop()
        self.obj_ids = list(TEST_SPLITS[LABEL_SPLIT[self.dataset]].obj_ids)
        label_of = {o: i for i, o in enumerate(self.obj_ids)}
        th, tw = cfg.train_img_size
        self.images = []
        for n in names:
            sp = TRAIN_SPLITS[n]
            H, W = sp.hw
            r = min(th / H, tw / W)
            root = os.path.join(datasets_root, "BOP_DATASETS", sp.dataset, sp.split)
            if not os.path.isdir(root):
                raise GdrnError(f"DATASETS.TRAIN {n}: {root} does not exist")
            for scene in sorted(int(d) for d in os.listdir(root) if d.isdigit()):
                sdir = os.path.join(root, "{:06d}".format(scene))
                gt, info = _load_json(os.path.join(sdir, "scene_gt.json")), _load_json(os.path.join(sdir, "scene_gt_info.json"))
                for im_id in sorted(gt, key=int):
                    rows, n_inst = [], 0
                    for k, g in enumerate(gt[im_id]):
                        if int(g["obj_id"]) not in label_of:
                            continue
                        inf = info[im_id][k]
                        if sp.filter_invalid and (inf["bbox_visib"][2] <= 1 or inf["bbox_visib"][3] <= 1):
                            continue
                        if sp.mask_value * int(inf["px_count_visib"]) < sp.min_area:
                            continue
                        n_inst += 1
                        x, y, w, h = inf["bbox_obj"]
                        x1, y1, x2, y2 = max(x, 0), max(y, 0), min(x + w, W), min(y + h, H)
                        if (x2 - x1) * (y2 - y1) > 0 and x2 >= x1 and y2 >= y1:
                            rows.append([x1, y1, x2, y2, label_of[int(g["obj_id"])]])
                    if n_inst == 0:   # the registrar drops an image without instances
                        continue
                    labels = np.zeros((len(rows), 5))
                    if rows:
                        labels[:] = rows
                    labels[:, :4] *= r
                    self.images.append({"path": os.path.join(sdir, "rgb", "{:06d}{}".format(int(im_id), sp.ext)),
                                        "hw": (H, W), "labels": labels, "image_id": int(im_id),
                                        "scene_im_id": f"{scene}/{int(im_id)}"})
        if not self.images:
            raise GdrnError(f"DATASETS.TRAIN {names}: no training images after filtering")
        self.with_labels = np.array([len(im["labels"]) > 0 for im in self.images])
        if not self.with_labels.any():
            raise GdrnError(f"DATASETS.TRAIN {names}: no image has a box (mixup draws until it finds one)")

    def __len__(self):
        return len(self.images)


# --------------------------------------------------------------------------------------------- box arithmetic
def mosaic_coordinate(i, xc, yc, w, h, input_h, input_w):
    """get_mosaic_coordinate -> (x1, y1, x2, y2) in the mosaic, (x1, y1, x2, y2) in the tile."""
    if i == 0:
        x1, y1, x2, y2 = max(xc - w, 0), max(yc - h, 0), xc, yc
        return (x1, y1, x2, y2), (w - (x2 - x1), h - (y2 - y1), w, h)
    if i == 1:
        x1, y1, x2, y2 = xc, max(yc - h, 0), min(xc + w, input_w * 2), yc
        return (x1, y1, x2, y2), (0, h - (y2 - y1), min(w, x2 - x1), h)
    if i == 2:
        x1, y1, x2, y2 = max(xc - w, 0), yc, xc, min(input_h * 2, yc + h)
        return (x1, y1, x2, y2), (w - (x2 - x1), 0, w, min(y2 - y1, h))
    x1, y1, x2, y2 = xc, yc, min(xc + w, input_w * 2), min(input_h * 2, yc + h)
    return (x1, y1, x2, y2), (0, 0, min(w, x2 - x1), min(y2 - y1, h))


def _xyxy2cxcywh(b):
    b[:, 2] = b[:, 2] - b[:, 0]
    b[:, 3] = b[:, 3] - b[:, 1]
    b[:, 0] = b[:, 0] + b[:, 2] * 0.5
    b[:, 1] = b[:, 1] + b[:, 3] * 0.5
    return b


def tile_size(ts, j, input_h, input_w):
    """(h, w, scale) of image j as a mosaic tile: load_resized_img's size, then the mosaic's own resize of it."""
    h1, w1, _ = letterbox_size(*ts.images[j]["hw"], input_h, input_w)
    scale = min(1.0 * input_h / h1, 1.0 * input_w / w1)
    return int(h1 * scale), int(w1 * scale), scale


class Sampler:
    """Draws the records of a batch and computes their targets: MosaicDetection.__getitem__'s randomness and box
    arithmetic for each sample, in the reference's order."""

    def __init__(self, cfg, ts):
        self.ts = ts
        self.w = cfg.aug_wrapper
        self.input_h, self.input_w = cfg.train_img_size
        self.color_prob = float(self.w["COLOR_AUG_PROB"])
        self.ops, self.random_order = ([], False)
        if self.color_prob > 0:
            self.ops, self.random_order = parse_color_aug(str(self.w["COLOR_AUG_CODE"]))
        self.S = max(len(self.ops), 1)
        drop = [op for op in self.ops if op["kind"] == "CoarseDropout"]
        # the colour program runs on the (w, h, c) transpose: the grid is round(W p) x round(H p)
        self.cell_hw = dropout_grid(drop[0], self.input_w, self.input_h) if drop else (1, 1)

    def empty(self, n):
        S, (ch, cw) = self.S, self.cell_hw
        return {"index": np.zeros((n, 4), np.int64), "mosaic": np.zeros(n, np.int32), "center": np.zeros((n, 2), np.int64),
                "affine": np.zeros((n, 6), np.float64), "mixup": np.zeros(n, np.int32), "jit": np.ones(n, np.float64),
                "mixup_flip": np.zeros(n, np.int32), "cp_index": np.zeros(n, np.int64), "offset": np.zeros((n, 2), np.int64),
                "t_on": np.zeros(n, np.int32), "t_hsv": np.zeros(n, np.int32), "t_gain": np.ones((n, 3), np.float64),
                "t_flip": np.zeros(n, np.int32), "fallback": np.zeros(n, np.int32),
                "w_hsv": np.zeros(n, np.int32), "w_gain": np.ones((n, 3), np.float64),
                "do_color": np.zeros(n, np.int32), "perm": np.tile(np.arange(S, dtype=np.int32), (n, 1)),
                "kind_at": np.full((n, S), -1, np.int32), "fpar": np.zeros((n, S, N_FPAR), np.float32),
                "ipar": np.zeros((n, S, N_IPAR), np.int32), "cells": np.ones((n, ch, cw), np.uint8),
                "targets": np.zeros((n, MAX_LABELS, 5), np.float32)}

    def draw(self, rng, n, mosaic_on=True):
        """-> record dict with a leading sample axis n (targets included)."""
        r = self.empty(n)
        for b in range(n):
            self._one(rng, r, b, mosaic_on)
        return r

    def _one(self, rng, r, b, mosaic_on):
        ts, w, ih, iw = self.ts, self.w, self.input_h, self.input_w
        N = len(ts)
        idx = int(rng.integers(N))
        r["index"][b, 0] = idx
        gate = rng.random() < float(w["mosaic_prob"])
        if bool(w["mosaic"]) and mosaic_on and gate:
            r["mosaic"][b] = 1
            yc = int(rng.uniform(0.5 * ih, 1.5 * ih))
            xc = int(rng.uniform(0.5 * iw, 1.5 * iw))
            r["center"][b] = (xc, yc)
            for k in range(1, 4):
                r["index"][b, k] = int(rng.integers(N))
            parts = []
            for i in range(4):
                j = int(r["index"][b, i])
                h, wd, scale = tile_size(ts, j, ih, iw)
                (lx1, ly1, _, _), (sx1, sy1, _, _) = mosaic_coordinate(i, xc, yc, wd, h, ih, iw)
                padw, padh = lx1 - sx1, ly1 - sy1
                src = ts.images[j]["labels"]
                lab = src.copy()
                if src.size > 0:
                    lab[:, 0] = scale * src[:, 0] + padw
                    lab[:, 1] = scale * src[:, 1] + padh
                    lab[:, 2] = scale * src[:, 2] + padw
                    lab[:, 3] = scale * src[:, 3] + padh
                parts.append(lab)
            labels = np.concatenate(parts, 0)
            np.clip(labels[:, 0], 0, 2 * iw, out=labels[:, 0])
            np.clip(labels[:, 1], 0, 2 * ih, out=labels[:, 1])
            np.clip(labels[:, 2], 0, 2 * iw, out=labels[:, 2])
            np.clip(labels[:, 3], 0, 2 * ih, out=labels[:, 3])
            # random_affine: get_affine_matrix's draws, then apply_affine_to_bboxes
            angle = _aug_param(rng, w["degrees"])
            scale = _aug_param(rng, w["mosaic_scale"], center=1.0)
            if scale <= 0.0:
                raise GdrnError("dataloader.train.aug_wrapper.mosaic_scale drew a scale <= 0")
            shx, shy = _aug_param(rng, w["shear"]), _aug_param(rng, w["shear"])
            tx, ty = _aug_param(rng, w["translate"]), _aug_param(rng, w["translate"])
            r["affine"][b] = (angle, scale, shx, shy, tx, ty)
            if len(labels) > 0:
                labels = self._affine_boxes(labels, affine_matrix(angle, scale, shx, shy, tx, ty, (iw, ih)), iw, ih)
            if bool(w["enable_mixup"]) and len(labels) > 0 and rng.random() < float(w["mixup_prob"]):
                labels = self._mixup(rng, r, b, labels)
            image_hw = (ih, iw)
        else:
            labels = ts.images[idx]["labels"].copy()
            image_hw = letterbox_size(*ts.images[idx]["hw"], ih, iw)[:2]
        self._train_transform(rng, r, b, labels, image_hw)
        if r["mosaic"][b]:
            if rng.random() < float(w["AUG_HSV_PROB"]):
                r["w_hsv"][b] = 1
                r["w_gain"][b] = rng.uniform(-1, 1, 3) * [w["HSV_H"], w["HSV_S"], w["HSV_V"]] + 1
            if self.ops and rng.random() < self.color_prob:
                self._color(rng, r, b)

    @staticmethod
    def _affine_boxes(targets, M, tw, th):
        n = len(targets)
        corners = np.ones((4 * n, 3))
        corners[:, :2] = targets[:, [0, 1, 2, 3, 0, 3, 2, 1]].reshape(4 * n, 2)
        corners = (corners @ M.T).reshape(n, 8)
        xs, ys = corners[:, 0::2], corners[:, 1::2]
        new = np.concatenate((xs.min(1), ys.min(1), xs.max(1), ys.max(1))).reshape(4, n).T
        new[:, 0::2] = new[:, 0::2].clip(0, tw)
        new[:, 1::2] = new[:, 1::2].clip(0, th)
        targets[:, :4] = new
        return targets

    def _mixup(self, rng, r, b, origin):
        ts, ih, iw = self.ts, self.input_h, self.input_w
        jit = float(rng.uniform(*self.w["mixup_scale"]))
        flip = bool(rng.uniform(0, 1) > 0.5)
        while True:
            cp = int(rng.integers(len(ts)))
            if ts.with_labels[cp]:
                break
        h1, w1, _ = letterbox_size(*ts.images[cp]["hw"], ih, iw)
        ratio = min(ih / h1, iw / w1) * jit
        oh, ow = int(ih * jit), int(iw * jit)
        ph, pw = max(oh, ih), max(ow, iw)
        yoff = int(rng.integers(0, ph - ih)) if ph > ih else 0
        xoff = int(rng.integers(0, pw - iw)) if pw > iw else 0
        r["mixup"][b], r["jit"][b], r["mixup_flip"][b], r["cp_index"][b] = 1, jit, int(flip), cp
        r["offset"][b] = (xoff, yoff)
        cp_labels = ts.images[cp]["labels"]
        box = cp_labels[:, :4].copy()
        box[:, 0::2] = np.clip(box[:, 0::2] * ratio, 0, ow)
        box[:, 1::2] = np.clip(box[:, 1::2] * ratio, 0, oh)
        if flip:
            box[:, 0::2] = ow - box[:, 0::2][:, ::-1]
        box[:, 0::2] = np.clip(box[:, 0::2] - xoff, 0, iw)
        box[:, 1::2] = np.clip(box[:, 1::2] - yoff, 0, ih)
        return np.vstack((origin, np.hstack((box, cp_labels[:, 4:5].copy()))))

    def _train_transform(self, rng, r, b, targets, image_hw):
        """TrainTransform: HSV gate and gains, mirror, letterbox scale, the min(w, h) > 1 filter and its fallback."""
        p = self.w
        if len(targets) == 0:
            return
        r["t_on"][b] = 1
        boxes, labels = targets[:, :4].copy(), targets[:, 4].copy()
        boxes_o, labels_o = _xyxy2cxcywh(targets[:, :4].copy()), targets[:, 4].copy()
        if rng.random() < float(p["preproc.hsv_prob"]):
            r["t_hsv"][b] = 1
            r["t_gain"][b] = rng.uniform(-1, 1, 3) * [0.5, 0.5, 0.5] + 1
        h, w = image_hw
        if rng.random() < float(p["preproc.flip_prob"]):
            r["t_flip"][b] = 1
            boxes[:, 0::2] = w - boxes[:, 2::-2]
        ratio = min(self.input_h / h, self.input_w / w)
        boxes = _xyxy2cxcywh(boxes) * ratio
        keep = np.minimum(boxes[:, 2], boxes[:, 3]) > 1
        boxes_t, labels_t = boxes[keep], labels[keep]
        if len(boxes_t) == 0:
            r["fallback"][b] = 1
            boxes_t, labels_t = boxes_o * ratio, labels_o
        t = np.hstack((labels_t[:, None], boxes_t))[:MAX_LABELS]
        r["targets"][b] = 0
        r["targets"][b, :len(t)] = t

    def _color(self, rng, r, b):
        r["do_color"][b] = 1
        nops = len(self.ops)
        perm = rng.permutation(nops).astype(np.int32) if self.random_order else np.arange(nops, dtype=np.int32)
        r["perm"][b, :nops] = perm
        for c, op in enumerate(self.ops):
            if rng.random() < op["prob"]:
                kind, f, i, cells = _draw_op(rng, op, self.cell_hw)
                s = int(np.nonzero(perm == c)[0][0])
                r["kind_at"][b, s], r["fpar"][b, s], r["ipar"][b, s] = kind, f, i
                if cells is not None:
                    r["cells"][b] = cells


def roles(rec, b):
    """The images sample b reads, in order: the four mosaic indices and the copy-paste index, or its own index."""
    if rec["mosaic"][b]:
        return [int(j) for j in rec["index"][b]] + ([int(rec["cp_index"][b])] if rec["mixup"][b] else [])
    return [int(rec["index"][b, 0])]


def decode(ts, rec, bs):
    """Host decode of samples bs: per sample the list of BGR images of roles(), each checked against its registrar
    size."""
    out = []
    for b in bs:
        ims = []
        for j in roles(rec, b):
            im = read_bgr(ts.images[j]["path"])
            if im.shape[:2] != tuple(ts.images[j]["hw"]):
                raise GdrnError(f"{ts.images[j]['path']} is {im.shape[1]}x{im.shape[0]}, its registrar says "
                                f"{ts.images[j]['hw'][1]}x{ts.images[j]['hw'][0]}")
            ims.append(im)
        out.append(ims)
    return out


# --------------------------------------------------------------------------------------------- device pipeline
class PinnedStaging:
    """Two pinned host buffers used in turn for the decoded images of a batch, so that their copy to the device is
    asynchronous.  A buffer is refilled only after the copy that last read it has finished (its event), which lets
    batch k + 1 be staged while batch k's copy and kernels run."""

    def __init__(self):
        self.slots = [[None, None], [None, None]]
        self.k = 0

    def upload(self, parts, dev):
        """parts: flat uint8 arrays -> their concatenation on `dev`, copied on the current stream."""
        import torch

        slot = self.slots[self.k]
        self.k ^= 1
        if slot[1] is not None:
            slot[1].synchronize()
        nbytes = sum(p.size for p in parts)
        if slot[0] is None or slot[0].numel() < nbytes:
            slot[0] = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
        host = slot[0].numpy()
        pos = 0
        for p in parts:
            host[pos:pos + p.size] = p
            pos += p.size
        out = slot[0][:nbytes].to(dev, non_blocking=True)
        slot[1] = torch.cuda.Event()
        slot[1].record()
        return out


def build_images(sampler, rec, images, dev, stats=None, staging=None):
    """The device pipeline of one batch -> (imgs [n,3,h,w] f32, the u8 stages as a dict for tests).  staging: a
    PinnedStaging reused across batches (a fresh one when None)."""
    import torch

    L = _lib.lib()
    ts, ih, iw = sampler.ts, sampler.input_h, sampler.input_w
    n = len(rec["mosaic"])
    st = _lib.current_stream()
    plane = ih * iw * 3

    def up(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=False)

    def ev(name):
        if stats is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            stats.setdefault("events", []).append((name, e))

    ev("upload")
    # source pool (decoded), stage-1 pool (load_resized_img), pool B: work slots, then tiles / canvases / d1 copies
    src_parts, src_off, pos = [], [], 0
    for ims in images:
        src_off.append([])
        for im in ims:
            src_parts.append(im.reshape(-1))
            src_off[-1].append(pos)
            pos += im.size
    src_d = (staging or PinnedStaging()).upload(src_parts, dev)
    jobs1, jobs2 = [], []
    r1_pos, b_pos = 0, n * plane
    tile_info = np.zeros((n, 4, 8), np.int64)
    mix_par = np.zeros((n, 6), np.int64)
    pre = np.zeros((n, 5), np.int64)
    hsv1 = []
    for b in range(n):
        js = roles(rec, b)
        r1 = []
        for k, j in enumerate(js):
            H, W = ts.images[j]["hw"]
            h1, w1, _ = letterbox_size(H, W, ih, iw)
            jobs1.append([src_off[b][k], H, W, r1_pos, h1, w1, h1, w1])
            r1.append((r1_pos, h1, w1))
            r1_pos += h1 * w1 * 3
        if rec["mosaic"][b]:
            xc, yc = (int(v) for v in rec["center"][b])
            for i in range(4):
                off, h1, w1 = r1[i]
                h, w, _ = letterbox_size(h1, w1, ih, iw)
                jobs2.append([off, h1, w1, b_pos, h, w, h, w])
                (lx1, ly1, lx2, ly2), (sx1, sy1, _, _) = mosaic_coordinate(i, xc, yc, w, h, ih, iw)
                tile_info[b, i] = (lx1, ly1, lx2, ly2, lx1 - sx1, ly1 - sy1, w, b_pos)
                b_pos += h * w * 3
            if rec["mixup"][b]:
                off, h1, w1 = r1[4]
                h, w, _ = letterbox_size(h1, w1, ih, iw)
                jobs2.append([off, h1, w1, b_pos, h, w, ih, iw])
                jit = float(rec["jit"][b])
                mix_par[b] = (b_pos, int(ih * jit), int(iw * jit), rec["mixup_flip"][b], rec["offset"][b, 0],
                              rec["offset"][b, 1])
                b_pos += plane
            pre[b] = (b * plane, ih, iw, 0, 1)
        else:
            off, h1, w1 = r1[0]
            jobs2.append([off, h1, w1, b_pos, h1, w1, h1, w1])
            pre[b] = (b_pos, h1, w1, 0, 0)
            b_pos += h1 * w1 * 3
        on = rec["t_on"][b] and not rec["fallback"][b]
        pre[b, 3] = int(on and rec["t_flip"][b])
        if on and rec["t_hsv"][b]:
            hsv1.append((b, pre[b, 0], pre[b, 1] * pre[b, 2]))
    r1_d = torch.empty(max(r1_pos, 1), dtype=torch.uint8, device=dev)
    pool = torch.empty(b_pos, dtype=torch.uint8, device=dev)
    jobs1_d, jobs2_d = up(np.asarray(jobs1, np.int64)), up(np.asarray(jobs2, np.int64))
    ev("resize")
    _lib.check(L.yolox_train_resize(_lib.ptr(src_d), _lib.ptr(r1_d), _lib.ptr(jobs1_d), len(jobs1),
                                    max(j[6] * j[7] for j in jobs1), st), "yolox_train_resize")
    _lib.check(L.yolox_train_resize(_lib.ptr(r1_d), _lib.ptr(pool), _lib.ptr(jobs2_d), len(jobs2),
                                    max(j[6] * j[7] for j in jobs2), st), "yolox_train_resize")
    mos = np.nonzero(rec["mosaic"])[0].astype(np.int32)
    ev("mosaic_affine")
    if len(mos):
        M = np.stack([affine_matrix(*rec["affine"][b], (iw, ih)).reshape(-1) for b in mos])
        ti_d, M_d, sel_d = up(tile_info[mos]), up(M), up(mos)
        _lib.check(L.yolox_train_mosaic_affine(_lib.ptr(pool), _lib.ptr(ti_d), _lib.ptr(M_d), _lib.ptr(sel_d), len(mos),
                                               ih, iw, _lib.ptr(pool), st), "yolox_train_mosaic_affine")
    mix = np.nonzero(rec["mixup"])[0].astype(np.int32)
    ev("mixup")
    if len(mix):
        mp_d, msel_d = up(mix_par[mix]), up(mix)
        _lib.check(L.yolox_train_mixup(_lib.ptr(pool), _lib.ptr(pool), _lib.ptr(mp_d), _lib.ptr(msel_d), len(mix), ih, iw,
                                       st), "yolox_train_mixup")
    ev("hsv_transform")
    if hsv1:
        ent = np.array([(o, p) for _, o, p in hsv1], np.int64)
        luts = np.stack([hsv_luts(rec["t_gain"][b]) for b, _, _ in hsv1])
        ent_d, lut_d = up(ent), up(luts)
        _lib.check(L.yolox_train_hsv(_lib.ptr(pool), _lib.ptr(ent_d), _lib.ptr(lut_d), len(hsv1), int(ent[:, 1].max()), 0, st),
                   "yolox_train_hsv")
    stages = {"pool": pool, "pre": pre}
    ev("preproc")
    P = torch.empty((n, ih, iw, 3), dtype=torch.uint8, device=dev)
    pre_d = up(pre)
    _lib.check(L.yolox_train_preproc(_lib.ptr(pool), _lib.ptr(pre_d), n, ih, iw, _lib.ptr(P), st), "yolox_train_preproc")
    ev("hsv_wrapper")
    wsel = [b for b in range(n) if rec["mosaic"][b] and rec["w_hsv"][b]]
    if wsel:
        ent_d = up(np.array([(b * plane, ih * iw) for b in wsel], np.int64))
        lut_d = up(np.stack([hsv_luts(rec["w_gain"][b]) for b in wsel]))
        rgb = int(str(sampler.w["FORMAT"]) == "RGB")
        _lib.check(L.yolox_train_hsv(_lib.ptr(P), _lib.ptr(ent_d), _lib.ptr(lut_d), len(wsel), ih * iw, rgb, st),
                   "yolox_train_hsv")
    ev("color")
    kind_at = np.where((rec["do_color"] > 0)[:, None], rec["kind_at"], -1).astype(np.int32)
    if (kind_at >= 0).any():
        S = kind_at.shape[1]
        ch, cw = rec["cells"].shape[1:]
        kind_d, fpar_d, ipar_d, cells_d = up(kind_at), up(rec["fpar"]), up(rec["ipar"]), up(rec["cells"])
        sums = torch.zeros(n, dtype=torch.int64, device=dev)
        Q = torch.empty_like(P)
        Ht, Wt = iw, ih   # the transposed layout: rows are the image's columns
        for s in range(S):
            if (kind_at[:, s] < 0).all():
                continue
            if (kind_at[:, s] == COLOR_OPS["EnhanceContrast"]).any():
                _lib.check(L.gdrn_train_luma_sum(_lib.ptr(P), n, Ht, Wt, _lib.ptr(kind_d), S, s, _lib.ptr(sums), st),
                           "gdrn_train_luma_sum")
            _lib.check(L.gdrn_train_color_step(_lib.ptr(P), _lib.ptr(Q), n, Ht, Wt, _lib.ptr(kind_d), _lib.ptr(fpar_d),
                                               _lib.ptr(ipar_d), S, s, _lib.ptr(cells_d), ch, cw, _lib.ptr(sums), st),
                       "gdrn_train_color_step")
            P, Q = Q, P
    ev("pack")
    out = torch.empty((n, 3, ih, iw), dtype=torch.float32, device=dev)
    tr_d = up(rec["mosaic"].astype(np.int32))
    _lib.check(L.yolox_train_pack(_lib.ptr(P), _lib.ptr(tr_d), n, ih, iw, _lib.ptr(out), st), "yolox_train_pack")
    ev("end")
    stages["final_u8"] = P
    return out, stages


class YoloxTrainBatcher:
    """Iterator over training batches (imgs [B,3,640,640] f32 on the device, targets [B,120,5] f32 (cls, cx, cy, w, h),
    img_info (two int64 tensors [B]), img_id [B,1] int64), as build_yolox_train_loader yields them.  Batch k draws its
    records from numpy.random.default_rng([seed, 2000 + k]); the last batch's records are kept in ``last_records``.
    ``close_mosaic()`` switches to the non-mosaic branch, as the trainer does for the last train.no_aug_epochs."""

    def __init__(self, cfg, datasets_root, *, seed=0, batch_size=None, device="cuda", num_workers=8):
        import torch

        check_train_config(cfg)
        self.cfg, self.seed = cfg, int(seed)
        self.batch_size = int(batch_size or cfg.train_total_batch_size)
        self.device = torch.device(device)
        self.ts = YoloxTrainSet(cfg, datasets_root)
        self.sampler = Sampler(cfg, self.ts)
        self.pool = ThreadPoolExecutor(max(1, num_workers))
        self.mosaic = True
        self.k = 0
        self.pending = None
        self.last_records = None
        self.stats = None   # a dict here collects the stage events of the next batch (bench_yolox_train_batch.py)
        self.staging = PinnedStaging()

    def close_mosaic(self):
        self.mosaic = False
        self.pending = None

    def _draw(self, k):
        rng = np.random.default_rng([self.seed, 2000 + k])
        rec = self.sampler.draw(rng, self.batch_size, self.mosaic)
        parts = max(1, min(self.batch_size, self.pool._max_workers))
        futs = [self.pool.submit(decode, self.ts, rec, c) for c in np.array_split(np.arange(self.batch_size), parts)]
        return rec, futs

    def __iter__(self):
        return self

    def __next__(self):
        import torch

        if self.pending is None:
            self.pending = self._draw(self.k)
        rec, futs = self.pending
        images = [ims for f in futs for ims in f.result()]
        self.k += 1
        self.pending = self._draw(self.k)   # the next batch decodes while this one runs on the GPU
        with torch.cuda.device(self.device):
            imgs, _ = build_images(self.sampler, rec, images, self.device, self.stats, self.staging)
        self.last_records = rec
        return (imgs, torch.from_numpy(rec["targets"].copy()).to(self.device),) + batch_info(self.ts, rec, self.sampler)

    def close(self):
        self.pool.shutdown(wait=True)


def batch_info(ts, rec, sampler):
    """(img_info, img_id) as default_collate stacks them: a mosaic sample reports (mix_img.shape[1], mix_img.shape[0])
    of its CHW image, (h, 3), and the image id of its last tile; any other sample (height, width) of its registrar and
    its own image id."""
    import torch

    n = len(rec["mosaic"])
    a, c, ids = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros((n, 1), np.int64)
    for b in range(n):
        if rec["mosaic"][b]:
            a[b], c[b] = sampler.input_h, 3
            ids[b, 0] = ts.images[int(rec["index"][b, 3])]["image_id"]
        else:
            j = int(rec["index"][b, 0])
            a[b], c[b] = ts.images[j]["hw"]
            ids[b, 0] = ts.images[j]["image_id"]
    return (torch.from_numpy(a), torch.from_numpy(c)), torch.from_numpy(ids)
