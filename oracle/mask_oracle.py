"""Restatements the save-results masks and the mask tools are checked against:

  * pycocotools' rleEncode / rleToString / rleFrString / rleDecode (maskApi.c), in NumPy / Python;
  * detectron2's GPU paste (paste_masks_in_image -> _do_paste_mask with skip_empty=False, F.grid_sample, >= threshold)
    as torch ops, on whatever device the inputs live on;
  * get_out_mask (engine_utils.py) for the mask probabilities;
  * the mask tools' metrics: compute_mean_iou (compute_mIoU_mask.py) and sklearn's binary f1_score.
"""
import numpy as np
import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------ pycocotools RLE
def rle_encode(mask):
    """[H,W] mask -> run lengths in column-major order, starting with the zero run (0 first when pixel (0,0) is set)."""
    flat = np.asarray(mask).astype(bool).ravel(order="F")
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(bounds).tolist()
    if flat.size and flat[0]:
        counts = [0] + counts
    return [int(c) for c in counts]


def rle_to_string(counts):
    """rleToString: for i > 2 the count minus cnts[i-2]; 5-bit groups from the low end, 0x20 = more follows, a final group
    with 0x10 set stands for a negative remainder; each char + 48."""
    out = []
    for i, c in enumerate(counts):
        x = int(c) - (int(counts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            g = x & 0x1F
            x >>= 5
            more = (x != -1) if (g & 0x10) else (x != 0)
            if more:
                g |= 0x20
            out.append(chr(g + 48))
    return "".join(out)


def rle_fr_string(s):
    """rleFrString: the string -> counts."""
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = ord(s[p]) - 48
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return counts


def rle_decode(counts, h, w):
    """rleDecode: counts -> uint8 [h,w] (runs alternate 0, 1, 0, ... in column-major order)."""
    if sum(counts) != h * w:
        raise ValueError(f"counts sum to {sum(counts)}, not {h * w}")
    vals = np.arange(len(counts)) % 2
    return np.repeat(vals, counts).astype(np.uint8).reshape((w, h)).T.copy()


def encode(mask):
    """binary_mask_to_rle(mask, compressed=True): {"size": [H, W], "counts": str}."""
    m = np.asarray(mask)
    return {"size": [int(m.shape[0]), int(m.shape[1])], "counts": rle_to_string(rle_encode(m))}


def decode(rle):
    return rle_decode(rle_fr_string(rle["counts"]), *rle["size"])


# ------------------------------------------------------------------------------------------------ detectron2 paste
def get_out_mask(pred_mask, mask_loss_type="L1"):
    bs = pred_mask.shape[0]
    if mask_loss_type == "L1":
        mx = torch.max(pred_mask.view(bs, -1), dim=-1)[0].view(bs, 1, 1, 1)
        mn = torch.min(pred_mask.view(bs, -1), dim=-1)[0].view(bs, 1, 1, 1)
        return (pred_mask - mn) / (mx - mn)
    if mask_loss_type in ("BCE", "RW_BCE", "dice"):
        return torch.sigmoid(pred_mask)
    raise NotImplementedError(mask_loss_type)


def paste_masks(masks, boxes, image_shape, threshold=0.5):
    """paste_masks_in_image on a GPU device: masks [N,M,M] probabilities, boxes [N,4] XYXY float32 -> bool [N,H,W].
    Every pixel is sampled (skip_empty=False); one torch op per step."""
    H, W = int(image_shape[0]), int(image_shape[1])
    dev = masks.device
    N = masks.shape[0]
    if N == 0:
        return torch.zeros((0, H, W), dtype=torch.bool, device=dev)
    x0, y0, x1, y1 = torch.split(boxes.to(torch.float32), 1, dim=1)
    img_y = torch.arange(0, H, device=dev, dtype=torch.float32) + 0.5
    img_x = torch.arange(0, W, device=dev, dtype=torch.float32) + 0.5
    img_y = (img_y - y0) / (y1 - y0) * 2 - 1
    img_x = (img_x - x0) / (x1 - x0) * 2 - 1
    gx = img_x[:, None, :].expand(N, H, W)
    gy = img_y[:, :, None].expand(N, H, W)
    grid = torch.stack([gx, gy], dim=3)
    out = F.grid_sample(masks[:, None].to(torch.float32), grid, mode="bilinear", padding_mode="zeros",
                        align_corners=False)[:, 0]
    return out >= threshold


def inst_rois(roi_center, scale):
    """The reference's inst_rois boxes: roi_center -/+ scale / 2 in float32 -> [n,4] XYXY."""
    n = roi_center.shape[0]
    return torch.cat([roi_center - scale.view(n, -1) / 2, roi_center + scale.view(n, -1) / 2], dim=1)


# ------------------------------------------------------------------------------------------------ mask metrics
def compute_mean_iou(pred, label):
    """compute_mIoU_mask.py: mean over the labels present in the GT of I / U."""
    pred, label = np.asarray(pred).ravel(), np.asarray(label).ravel()
    ious = []
    for val in np.unique(label):
        p, g = pred == val, label == val
        ious.append(float(np.sum(p & g)) / float(np.sum(p | g)))
    return float(np.mean(ious))


def f1_binary(pred, label):
    """sklearn f1_score(label, pred) for binary labels: 2 TP / (2 TP + FP + FN), 0 when that is 0 / 0."""
    p, g = np.asarray(pred).ravel().astype(bool), np.asarray(label).ravel().astype(bool)
    tp, fp, fn = int(np.sum(p & g)), int(np.sum(p & ~g)), int(np.sum(~p & g))
    d = 2 * tp + fp + fn
    return 2.0 * tp / d if d else 0.0
