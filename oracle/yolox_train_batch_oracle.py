"""NumPy / cv2 restatement of MosaicDetection.__getitem__ (det/yolox/data/datasets/mosaicdetection.py) with its mixup,
TrainTransform, preproc and augment_hsv (det/yolox/data/data_augment.py), driven by the records of
gdrnpp_bop2022_b200.yolox_train_batch, and of the detector's registrars + Base_DatasetFromList.load_anno, which read
the mask PNGs as the reference does.  The box arithmetic is restated here on its own; the colour program comes from
oracle/train_batch_oracle.py.  Tests compare the CUDA pipeline with it bit for bit (images) and within 1e-6 (targets)."""
import json
import math
import os

import cv2
import numpy as np

from oracle import train_batch_oracle as TBO

MAX_LABELS = 120


# --------------------------------------------------------------------------------------------- registrars
def _bool_area_lt30(m):   # lm_pbr.py, itodd_pbr.py, tudl_pbr.py: mask_single.astype("bool").sum() < 30
    return m.astype("bool").sum() < 30


def _raw_area_lt30(m):   # tless_pbr.py, icbin_pbr.py, tudl_train_real.py: the raw PNG's sum < 30
    return m.sum() < 30


def _raw_area_le64(m):   # hb_pbr.py, ycbv_pbr.py, tless_primesense_train.py: the raw PNG's sum <= 64
    return m.sum() <= 64


# name -> (dataset dir, split dir, image ext, (height, width), dropped-by-area, filter_invalid)
REGISTRARS = {
    "lmo_pbr_train": ("lmo", "train_pbr", ".jpg", (480, 640), _bool_area_lt30, True),
    "tless_pbr_train": ("tless", "train_pbr", ".jpg", (540, 720), _raw_area_lt30, False),
    "tudl_pbr_train": ("tudl", "train_pbr", ".jpg", (480, 640), _bool_area_lt30, True),
    "icbin_pbr_train": ("icbin", "train_pbr", ".jpg", (480, 640), _raw_area_lt30, False),
    "itodd_pbr_train": ("itodd", "train_pbr", ".jpg", (960, 1280), _bool_area_lt30, True),
    "hb_pbr_train": ("hb", "train_pbr", ".jpg", (480, 640), _raw_area_le64, True),
    "ycbv_train_pbr": ("ycbv", "train_pbr", ".jpg", (480, 640), _raw_area_le64, True),
    "tless_primesense_train": ("tless", "train_primesense", ".png", (400, 400), _raw_area_le64, True),
    "tudl_train_real": ("tudl", "train_real", ".png", (480, 640), _raw_area_lt30, True),
}


def registrar_images(datasets_root, name, obj_ids, size=(640, 640)):
    """The registrar's records of one split, then load_anno -> [(rgb path, labels [k,5])] in scene / image order.
    Each instance's visible area comes from its mask_visib PNG read unchanged, as the registrar reads it."""
    ds, split, ext, (H, W), dropped, filter_invalid = REGISTRARS[name]
    root = os.path.join(datasets_root, "BOP_DATASETS", ds, split)
    out = []
    for scene in sorted(int(d) for d in os.listdir(root) if d.isdigit()):
        sdir = os.path.join(root, "{:06d}".format(scene))
        with open(os.path.join(sdir, "scene_gt.json")) as f:
            gt_dict = json.load(f)
        with open(os.path.join(sdir, "scene_gt_info.json")) as f:
            info_dict = json.load(f)
        for str_im_id in gt_dict:
            insts = []
            for anno_i, anno in enumerate(gt_dict[str_im_id]):
                if anno["obj_id"] not in obj_ids:
                    continue
                info = info_dict[str_im_id][anno_i]
                _, _, w, h = info["bbox_visib"]
                if filter_invalid and (h <= 1 or w <= 1):
                    continue
                m = cv2.imread(os.path.join(sdir, "mask_visib", "{:06d}_{:06d}.png".format(int(str_im_id), anno_i)),
                               cv2.IMREAD_UNCHANGED)
                if dropped(m):
                    continue
                insts.append((obj_ids.index(anno["obj_id"]), info["bbox_obj"]))
            if not insts:
                continue
            # load_anno: XYWH -> XYXY, clipped to the registrar's size, area > 0, scaled to the training size
            rows = []
            for cls, (x, y, w, h) in insts:
                x1, y1, x2, y2 = np.max((x, 0)), np.max((y, 0)), np.min((x + w, W)), np.min((y + h, H))
                if (x2 - x1) * (y2 - y1) > 0 and x2 >= x1 and y2 >= y1:
                    rows.append((x1, y1, x2, y2, cls))
            res = np.zeros((len(rows), 5))
            for i, r in enumerate(rows):
                res[i] = r
            res[:, :4] *= min(size[0] / H, size[1] / W)
            out.append((os.path.join(sdir, "rgb", "{:06d}{}".format(int(str_im_id), ext)), res))
    return out


def load_resized(img, size):
    r = min(size[0] / img.shape[0], size[1] / img.shape[1])
    return cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR).astype(np.uint8)


def affine(a, size):
    """get_affine_matrix from the record's (angle, scale, shear_x, shear_y, tx, ty)."""
    angle, scale, shx, shy, tx, ty = (float(v) for v in a)
    R = cv2.getRotationMatrix2D(angle=angle, center=(0, 0), scale=scale)
    M = np.ones([2, 3])
    M[0] = R[0] + math.tan(shy * math.pi / 180) * R[1]
    M[1] = R[1] + math.tan(shx * math.pi / 180) * R[0]
    M[0, 2], M[1, 2] = tx * size[0], ty * size[1]
    return M


def augment_hsv(img, gains, source_format):
    """augment_hsv with the drawn gains r, in place."""
    code = (cv2.COLOR_RGB2HSV, cv2.COLOR_HSV2RGB) if source_format == "RGB" else (cv2.COLOR_BGR2HSV, cv2.COLOR_HSV2BGR)
    hue, sat, val = cv2.split(cv2.cvtColor(img, code[0]))
    x = np.arange(0, 256, dtype=np.int16)
    lut_hue = ((x * gains[0]) % 180).astype(np.uint8)
    lut_sat = np.clip(x * gains[1], 0, 255).astype(np.uint8)
    lut_val = np.clip(x * gains[2], 0, 255).astype(np.uint8)
    hsv = cv2.merge((cv2.LUT(hue, lut_hue), cv2.LUT(sat, lut_sat), cv2.LUT(val, lut_val))).astype(np.uint8)
    cv2.cvtColor(hsv, code[1], dst=img)


def preproc(img, size):
    padded = np.ones((size[0], size[1], 3), dtype=np.uint8) * 114
    r = min(size[0] / img.shape[0], size[1] / img.shape[1])
    resized = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR).astype(np.uint8)
    padded[: int(img.shape[0] * r), : int(img.shape[1] * r)] = resized
    return np.ascontiguousarray(padded.transpose(2, 0, 1), dtype=np.float32), r


def cxcywh(b):
    out = b.copy()
    out[:, 2] = b[:, 2] - b[:, 0]
    out[:, 3] = b[:, 3] - b[:, 1]
    out[:, 0] = b[:, 0] + out[:, 2] * 0.5
    out[:, 1] = b[:, 1] + out[:, 3] * 0.5
    return out


def mosaic(rec, b, ims, labels_of, size):
    ih, iw = size
    xc, yc = (int(v) for v in rec["center"][b])
    canvas = np.full((ih * 2, iw * 2, 3), 114, dtype=np.uint8)
    boxes = []
    for i in range(4):
        img = load_resized(ims[i], size)
        h0, w0 = img.shape[:2]
        s = min(1.0 * ih / h0, 1.0 * iw / w0)
        img = cv2.resize(img, (int(w0 * s), int(h0 * s)), interpolation=cv2.INTER_LINEAR)
        h, w = img.shape[:2]
        if i == 0:
            L = (max(xc - w, 0), max(yc - h, 0), xc, yc)
            S = (w - (L[2] - L[0]), h - (L[3] - L[1]), w, h)
        elif i == 1:
            L = (xc, max(yc - h, 0), min(xc + w, iw * 2), yc)
            S = (0, h - (L[3] - L[1]), min(w, L[2] - L[0]), h)
        elif i == 2:
            L = (max(xc - w, 0), yc, xc, min(ih * 2, yc + h))
            S = (w - (L[2] - L[0]), 0, w, min(L[3] - L[1], h))
        else:
            L = (xc, yc, min(xc + w, iw * 2), min(ih * 2, yc + h))
            S = (0, 0, min(w, L[2] - L[0]), min(L[3] - L[1], h))
        canvas[L[1]:L[3], L[0]:L[2]] = img[S[1]:S[3], S[0]:S[2]]
        lab = labels_of(int(rec["index"][b, i])).copy()
        if lab.size:
            lab[:, [0, 2]] = s * lab[:, [0, 2]] + (L[0] - S[0])
            lab[:, [1, 3]] = s * lab[:, [1, 3]] + (L[1] - S[1])
        boxes.append(lab)
    boxes = np.concatenate(boxes, 0)
    boxes[:, [0, 2]] = np.clip(boxes[:, [0, 2]], 0, 2 * iw)
    boxes[:, [1, 3]] = np.clip(boxes[:, [1, 3]], 0, 2 * ih)
    M = affine(rec["affine"][b], (iw, ih))
    img = cv2.warpAffine(canvas, M, dsize=(iw, ih), borderValue=(114, 114, 114))
    if len(boxes):
        n = len(boxes)
        pts = np.ones((4 * n, 3))
        pts[:, :2] = boxes[:, [0, 1, 2, 3, 0, 3, 2, 1]].reshape(4 * n, 2)
        pts = (pts @ M.T).reshape(n, 8)
        xs, ys = pts[:, 0::2], pts[:, 1::2]
        boxes[:, 0], boxes[:, 1] = xs.min(1).clip(0, iw), ys.min(1).clip(0, ih)
        boxes[:, 2], boxes[:, 3] = xs.max(1).clip(0, iw), ys.max(1).clip(0, ih)
    return img, boxes


def mixup(rec, b, img, boxes, cp_img, cp_labels, size):
    ih, iw = size
    jit, flip = float(rec["jit"][b]), bool(rec["mixup_flip"][b])
    xoff, yoff = (int(v) for v in rec["offset"][b])
    src = load_resized(cp_img, size)
    cp = np.ones((ih, iw, 3), dtype=np.uint8) * 114
    ratio = min(ih / src.shape[0], iw / src.shape[1])
    cp[: int(src.shape[0] * ratio), : int(src.shape[1] * ratio)] = cv2.resize(
        src, (int(src.shape[1] * ratio), int(src.shape[0] * ratio)), interpolation=cv2.INTER_LINEAR)
    cp = cv2.resize(cp, (int(cp.shape[1] * jit), int(cp.shape[0] * jit)))
    ratio *= jit
    if flip:
        cp = cp[:, ::-1, :]
    oh, ow = cp.shape[:2]
    padded = np.zeros((max(oh, ih), max(ow, iw), 3), dtype=np.uint8)
    padded[:oh, :ow] = cp
    crop = padded[yoff:yoff + ih, xoff:xoff + iw]
    bx = cp_labels[:, :4].copy()
    bx[:, 0::2] = np.clip(bx[:, 0::2] * ratio, 0, ow)
    bx[:, 1::2] = np.clip(bx[:, 1::2] * ratio, 0, oh)
    if flip:
        bx[:, [0, 2]] = ow - bx[:, [2, 0]]
    bx[:, 0::2] = np.clip(bx[:, 0::2] - xoff, 0, iw)
    bx[:, 1::2] = np.clip(bx[:, 1::2] - yoff, 0, ih)
    boxes = np.vstack((boxes, np.hstack((bx, cp_labels[:, 4:5]))))
    blended = 0.5 * img.astype(np.float32) + 0.5 * crop.astype(np.float32)
    return blended.astype(np.uint8), boxes


def train_transform(rec, b, image, targets, size):
    """-> (float32 CHW image, padded [120,5] targets)."""
    if len(targets) == 0:
        return preproc(image, size)[0], np.zeros((MAX_LABELS, 5), np.float32)
    image_o = image.copy()
    boxes_o = cxcywh(targets[:, :4])
    if rec["t_hsv"][b]:
        augment_hsv(image, rec["t_gain"][b], "BGR")
    boxes = targets[:, :4].copy()
    width = image.shape[1]
    if rec["t_flip"][b]:
        image = image[:, ::-1]
        boxes[:, [0, 2]] = width - targets[:, [2, 0]]
    out, r = preproc(image, size)
    boxes = cxcywh(boxes) * r
    keep = np.minimum(boxes[:, 2], boxes[:, 3]) > 1
    boxes_t, labels_t = boxes[keep], targets[keep, 4]
    if len(boxes_t) == 0:
        out, r_o = preproc(image_o, size)
        boxes_t, labels_t = boxes_o * r_o, targets[:, 4]
    t = np.hstack((labels_t[:, None], boxes_t))[:MAX_LABELS]
    padded = np.zeros((MAX_LABELS, 5))
    padded[:len(t)] = t
    return out, padded.astype(np.float32)


def replay(records, images, labels_of, size=(640, 640), source_format="RGB"):
    """records: yolox_train_batch's record dict; images[b]: the decoded BGR images of the sample's roles (mosaic: its
    four indices, then the copy-paste image when it mixes; otherwise its own image); labels_of(i): load_anno's
    [k,5] array of image i.  -> (imgs [n,3,h,w] f32, targets [n,120,5] f32)."""
    n = len(records["mosaic"])
    imgs = np.zeros((n, 3) + tuple(size), np.float32)
    targets = np.zeros((n, MAX_LABELS, 5), np.float32)
    for b in range(n):
        ims = images[b]
        if records["mosaic"][b]:
            img, boxes = mosaic(records, b, ims, labels_of, size)
            if records["mixup"][b]:
                img, boxes = mixup(records, b, img, boxes, ims[4], labels_of(int(records["cp_index"][b])), size)
            out, targets[b] = train_transform(records, b, img, boxes, size)
            t = out.transpose(2, 1, 0).astype(np.uint8).copy()
            if records["w_hsv"][b]:
                augment_hsv(t, records["w_gain"][b], source_format)
            if records["do_color"][b]:
                for s in range(records["kind_at"].shape[1]):
                    t = TBO.apply_op(t, records["kind_at"][b, s], records["fpar"][b, s], records["ipar"][b, s],
                                     records["cells"][b])
            imgs[b] = t.transpose(2, 1, 0).astype(np.float32)
        else:
            img = load_resized(ims[0], size)
            imgs[b], targets[b] = train_transform(records, b, img, labels_of(int(records["index"][b, 0])).copy(), size)
    return imgs, targets
