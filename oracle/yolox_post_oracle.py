"""NumPy restatement of the YOLOX post-process (det/yolox/utils/boxes.py:34-80 with YOLOXHead.decode_outputs, and the
keep-single-instance post-process of the reference predictor, predictor_yolo.py:84-140), one function per stage.

Each stage returns an fp64 value and, where the reference's fp32 rounding decides, an exact fp32 replica of what torch
and torchvision compute.  Three torchvision behaviours decide which boxes survive:
  * batched_nms on CUDA runs ``_batched_nms_coordinate_trick`` while ``boxes.numel() <= 100_000`` (n <= 25 000
    candidates): every box is shifted by ``cls * (max_coordinate + 1)`` in fp32 and one NMS runs over all boxes with
    no class check.  Above that it runs ``_batched_nms_vanilla``: one NMS per class on the unshifted boxes.
  * the sm_90 build of ``nms_kernel_impl<float>`` computes the later-ranked box's area inside an FMA:
    ``fma(bw, bh, Sa) - inter``, and compares with the threshold rounded to fp32 (iou_cuda_f32).
  * the CPU ``nms`` (the keep-single-instance path: its rows live on the host) rounds every product and compares the
    fp32 IoU with the double threshold (iou_cpu_f32).
Sorting is stable (descending score, then ascending index) everywhere here; tests that compare with torch's CUDA sort
say where that holds.
"""
from fractions import Fraction

import numpy as np

F32, F64 = np.float32, np.float64
TRICK_MAX_CANDIDATES = 25_000   # torchvision batched_nms on CUDA: coordinate trick while boxes.numel() <= 100_000


# ---------------------------------------------------------------------------------------------------------------------
# decode, class max, score and filter, compaction, rank
# ---------------------------------------------------------------------------------------------------------------------
def anchor_grid(hw, strides):
    """(gx, gy, stride) per anchor [A] for levels hw = [(rows, cols), ...] concatenated in order (row-major cells)."""
    gx, gy, st = [], [], []
    for (h, w), s in zip(hw, strides):
        yv, xv = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        gx.append(xv.ravel()); gy.append(yv.ravel()); st.append(np.full(h * w, s))
    return np.concatenate(gx), np.concatenate(gy), np.concatenate(st)


def decode(raw, hw, strides):
    """raw [A, >=4] fp32 head outputs -> (cxcy32 [A, 2] exact fp32 replica of (x + grid) * stride,
    wh64 [A, 2] = exp(w) * stride in fp64).  The fp32 w, h depend on the device's expf (within 2 ulp of wh64)."""
    gx, gy, st = anchor_grid(hw, strides)
    r = np.asarray(raw, F32)
    cx = ((r[:, 0] + gx.astype(F32)) * st.astype(F32)).astype(F32)
    cy = ((r[:, 1] + gy.astype(F32)) * st.astype(F32)).astype(F32)
    wh = np.exp(r[:, 2:4].astype(F64)) * st[:, None]
    return np.stack([cx, cy], 1), wh


def xyxy(cx, cy, w, h):
    """fp32 cxcywh -> fp32 (x1, y1, x2, y2) as torch computes ``cx - w / 2`` (both roundings)."""
    cx, cy, w, h = (np.asarray(v, F32) for v in (cx, cy, w, h))
    hw2, hh2 = (w / F32(2)).astype(F32), (h / F32(2)).astype(F32)
    return np.stack([cx - hw2, cy - hh2, cx + hw2, cy + hh2], -1).astype(F32)


def class_max(cls_scores):
    """[A, nc] -> (class_conf, class_pred): the first maximum, as torch.max."""
    c = np.asarray(cls_scores, F32)
    p = np.argmax(c, 1)
    return c[np.arange(len(c)), p], p


def score_filter(obj, cls_conf, conf):
    """-> (score32, keep32, keep64): score = obj * class_conf in fp32, kept when >= float32(conf) (torch compares a CUDA
    float tensor with the scalar rounded to fp32); keep64 decides on the exact product and the double threshold.
    Where keep32 != keep64 the rounding of the product (or of conf) decides: that is the fp64 band."""
    o, c = np.asarray(obj, F32), np.asarray(cls_conf, F32)
    s32 = (o * c).astype(F32)
    s64 = o.astype(F64) * c.astype(F64)   # exact: a product of two fp32 values fits a double
    return s32, s32 >= F32(conf), s64 >= conf


def compact(keep):
    """Ordered compaction: the indices boolean indexing keeps, in anchor order."""
    return np.nonzero(np.asarray(keep))[0]


def rank(score):
    """order[r] = candidate index of rank r: descending score, ties by ascending index (a stable sort)."""
    s = np.asarray(score, F32)
    return np.lexsort((np.arange(len(s)), -s.astype(F64)))


# ---------------------------------------------------------------------------------------------------------------------
# IoU in three forms; a is the earlier-ranked box
# ---------------------------------------------------------------------------------------------------------------------
def round_f32(q):
    """A Fraction rounded to the nearest fp32 (ties to even)."""
    r = F32(float(q))
    cands = [r, np.nextafter(r, F32(-np.inf)), np.nextafter(r, F32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))
    return F32(best)


def fma_f32(x, y, z):
    """fp32 fma(x, y, z) rounded once, exactly.  x * y is exact in fp64; TwoSum gives the rounding error of the fp64
    sum, which decides the one case double rounding gets wrong: an fp64 sum on an fp32 midpoint."""
    x, y, z = np.broadcast_arrays(np.asarray(x, F32), np.asarray(y, F32), np.asarray(z, F32))
    p, zz = x.astype(F64) * y.astype(F64), z.astype(F64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + zz
        bb = s - p
        err = (p - (s - bb)) + (zz - bb)
        r = s.astype(F32)
        t = r.astype(F64)
        other = np.nextafter(r, np.where(s > t, F32(np.inf), F32(-np.inf)).astype(F32))
        mid = (s != t) & np.isfinite(s) & (np.abs(s - t) == np.abs(other.astype(F64) - s))
        toward = mid & (err != 0) & (np.sign(err) == np.sign(s - t))
    return np.where(toward, other, r).astype(F32)


def fma_f32_fraction(x, y, z):
    """Scalar fma via exact rational arithmetic (pins fma_f32)."""
    return round_f32(Fraction(float(F32(x))) * Fraction(float(F32(y))) + Fraction(float(F32(z))))


def _overlap(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    w = np.maximum((np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0])).astype(F32), F32(0))
    h = np.maximum((np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1])).astype(F32), F32(0))
    return a, b, w, h


def iou64(a, b):
    """IoU in fp64 of boxes given in fp32 or fp64 (0/0 -> nan, which suppresses nothing)."""
    a, b = np.asarray(a, F64), np.asarray(b, F64)
    w = np.maximum(np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]), 0.0)
    h = np.maximum(np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]), 0.0)
    inter = w * h
    sa = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1])
    sb = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / (sa + sb - inter)


def iou_cuda_f32(a, b):
    """torchvision's sm_90 nms_kernel_impl<float>: Sa = FMUL, denominator = fma(b.x2 - b.x0, b.y3 - b.y1, Sa) - inter."""
    a, b, w, h = _overlap(a, b)
    inter = (w * h).astype(F32)
    sa = ((a[..., 2] - a[..., 0]).astype(F32) * (a[..., 3] - a[..., 1]).astype(F32)).astype(F32)
    den = (fma_f32((b[..., 2] - b[..., 0]).astype(F32), (b[..., 3] - b[..., 1]).astype(F32), sa) - inter).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (inter / den).astype(F32)


def iou_cpu_f32(a, b):
    """torchvision's CPU nms: every product and sum rounded on its own, (Sa + Sb) - inter."""
    a, b, w, h = _overlap(a, b)
    inter = (w * h).astype(F32)
    sa = ((a[..., 2] - a[..., 0]).astype(F32) * (a[..., 3] - a[..., 1]).astype(F32)).astype(F32)
    sb = ((b[..., 2] - b[..., 0]).astype(F32) * (b[..., 3] - b[..., 1]).astype(F32)).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (inter / ((sa + sb).astype(F32) - inter).astype(F32)).astype(F32)


def suppresses_cuda(iou32, thr):
    return iou32 > F32(thr)          # the double threshold converted to fp32, FSETP.GT


def suppresses_cpu(iou32, thr):
    return iou32.astype(F64) > thr   # the fp32 IoU promoted, compared with the double threshold


# ---------------------------------------------------------------------------------------------------------------------
# suppression masks, greedy reduce, the three NMS calls
# ---------------------------------------------------------------------------------------------------------------------
def trick_offsets(boxes, cls):
    """_batched_nms_coordinate_trick's fp32 shift: cls * (boxes.max() + 1) per box."""
    b = np.asarray(boxes, F32)
    mx = F32(b.max()) if b.size else F32(0)
    return (np.asarray(cls, F32) * F32(mx + F32(1))).astype(F32), mx


def suppress_matrix(sorted_boxes, thr, form="cuda", cls=None):
    """[n, n] bool, entry (i, j) for j > i: sorted box i suppresses sorted box j.  ``cls`` (sorted classes) adds the
    per-class check of the vanilla path; form "cuda" / "cpu" picks the IoU arithmetic."""
    b = np.asarray(sorted_boxes, F32)
    n = len(b)
    iou = (iou_cuda_f32 if form == "cuda" else iou_cpu_f32)(b[:, None, :], b[None, :, :])
    s = suppresses_cuda(iou, thr) if form == "cuda" else suppresses_cpu(iou, thr)
    s &= np.triu(np.ones((n, n), bool), 1)
    if cls is not None:
        c = np.asarray(cls)
        s &= c[:, None] == c[None, :]
    return s


def mask_words(sup, n_words=None):
    """Suppression matrix -> the kernel's bit masks [n, words] uint64 (bit k of word w: column w * 64 + k)."""
    n = sup.shape[0]
    words = n_words or (n + 63) // 64
    pad = np.zeros((n, words * 64), bool)
    pad[:, :n] = sup
    bits = pad.reshape(n, words, 64).astype(np.uint64) << np.arange(64, dtype=np.uint64)
    return np.bitwise_or.reduce(bits, axis=2)


def greedy(sup, max_out=None):
    """Greedy pass over a suppression matrix (sorted order) -> kept sorted positions, capped at max_out."""
    n = sup.shape[0]
    removed = np.zeros(n, bool)
    kept = []
    for i in range(n):
        if removed[i]:
            continue
        kept.append(i)
        removed |= sup[i]
    kept = np.array(kept, np.int64)
    return kept if max_out is None else kept[:max_out]


def greedy_words(words, n, max_out=None):
    """Greedy pass over the kernel's own bit masks [n, words] (sorted order) -> kept sorted positions."""
    w = np.asarray(words).view(np.uint64)
    bits = ((w[:, :, None] >> np.arange(64, dtype=np.uint64)) & np.uint64(1)).astype(bool).reshape(len(w), -1)[:n, :n]
    return greedy(np.triu(bits, 1), max_out)


def nms(boxes, scores, thr, form="cuda", cls=None):
    """torchvision.ops.nms (form "cuda" or "cpu") -> kept indices in descending score order; ``cls`` restricts
    suppression to equal classes (one NMS per class, merged by score: the vanilla batched path)."""
    order = rank(scores)
    c = None if cls is None else np.asarray(cls)[order]
    return order[greedy(suppress_matrix(np.asarray(boxes, F32)[order], thr, form, c))]


def batched_nms_trick(boxes, scores, cls, thr, form="cuda"):
    off, _ = trick_offsets(boxes, cls)
    return nms((np.asarray(boxes, F32) + off[:, None]).astype(F32), scores, thr, form)


def batched_nms_vanilla(boxes, scores, cls, thr, form="cuda"):
    return nms(boxes, scores, thr, form, cls)


def batched_nms(boxes, scores, cls, thr):
    """torchvision.ops.batched_nms on CUDA: the coordinate trick up to 25 000 boxes, vanilla above."""
    if len(boxes) <= TRICK_MAX_CANDIDATES:
        return batched_nms_trick(boxes, scores, cls, thr)
    return batched_nms_vanilla(boxes, scores, cls, thr)


def postprocess(dec, num_classes, conf, thr, class_agnostic=False, max_out=None):
    """boxes.postprocess for one image of decoded fp32 det_preds [A, 5 + nc] -> dict of every stage: boxes (xyxy fp32),
    score, keep, cand (compacted indices), order (ranked candidate positions), kept (rows of cand[order], capped)."""
    d = np.asarray(dec, F32)
    boxes = xyxy(d[:, 0], d[:, 1], d[:, 2], d[:, 3])
    cc, cp = class_max(d[:, 5:5 + num_classes])
    s32, keep, _ = score_filter(d[:, 4], cc, conf)
    cand = compact(keep)
    b, s, c = boxes[cand], s32[cand], cp[cand].astype(F32)
    order = rank(s)
    if class_agnostic:
        sb = b[order]
    elif len(cand) <= TRICK_MAX_CANDIDATES:
        off, _ = trick_offsets(b, c)
        sb = (b + off[:, None]).astype(F32)[order]
    else:
        sb = b[order]
    sup = suppress_matrix(sb, thr, "cuda", None if class_agnostic or len(cand) <= TRICK_MAX_CANDIDATES else c[order])
    kept = greedy(sup, max_out)
    rows = np.concatenate([b, d[cand, 4:5], cc[cand, None], c[:, None]], 1).astype(F32)
    return {"boxes": boxes, "score": s32, "keep": keep, "cand": cand, "order": order, "sup": sup,
            "kept": order[kept], "rows": rows[order[kept]]}


# ---------------------------------------------------------------------------------------------------------------------
# keep-single-instance (predictor_yolo.py:84-140, class_agnostic=True)
# ---------------------------------------------------------------------------------------------------------------------
def ksi_select(score32, cls_pred, keep, num_classes):
    """Per class the anchor the reference's loop picks: strictly greater than a running max that starts at 0, so the
    lowest anchor wins a tie and a score of 0 is never picked -> sel [nc] (-1 = none)."""
    sel = np.full(num_classes, -1, np.int64)
    best = np.zeros(num_classes, F32)
    for a in compact(keep):
        c = cls_pred[a]
        if score32[a] > best[c]:
            best[c], sel[c] = score32[a], a
    return sel


def keep_single_instance(dec, num_classes, conf, thr):
    """-> (sel [nc], rows [n, 7] fp32 in ascending class order): selection, torchvision's CPU nms over the selected rows
    (in class order, so equal scores keep the lower class), output sorted by class."""
    d = np.asarray(dec, F32)
    boxes = xyxy(d[:, 0], d[:, 1], d[:, 2], d[:, 3])
    cc, cp = class_max(d[:, 5:5 + num_classes])
    s32, keep, _ = score_filter(d[:, 4], cc, conf)
    sel = ksi_select(s32, cp, keep, num_classes)
    cls = np.nonzero(sel >= 0)[0]
    a = sel[cls]
    rows = np.concatenate([boxes[a], d[a, 4:5], cc[a, None], cls[:, None].astype(F32)], 1).astype(F32)
    k = nms(rows[:, :4], s32[a], thr, "cpu")
    return sel, rows[np.sort(k)]


# ---------------------------------------------------------------------------------------------------------------------
# planted near-threshold pairs
# ---------------------------------------------------------------------------------------------------------------------
def near_threshold_pairs(rng, n, thr, span=64, lo=20.0, hi=600.0):
    """Random box pairs in cxcywh fp32 whose IoU scans a band of +-span ulps of b's centre around the fp64 root of
    IoU = thr (b slides along x).  -> (pa [m, 4], pb [m, 4]) fp32 cxcywh, every scanned pair."""
    wa, ha = rng.uniform(20, 120, n), rng.uniform(20, 120, n)
    wb, hb = wa * rng.uniform(0.8, 1.25, n), ha * rng.uniform(0.8, 1.25, n)
    cxa, cya = rng.uniform(lo + 80, hi - 80, n), rng.uniform(lo + 80, hi - 80, n)
    dy = rng.uniform(-0.1, 0.1, n) * ha
    pa = np.stack([cxa, cya, wa, ha], 1).astype(F32)
    pb0 = np.stack([cxa, cya + dy, wb, hb], 1).astype(F32)

    def iou_at(d):
        pb = pb0.astype(F64).copy()
        pb[:, 0] += d
        return iou64(xyxy(*pa.T), xyxy(*pb.astype(F32).T))

    d_lo, d_hi = np.abs(wa - wb) / 2, (wa + wb) / 2
    ok = iou_at(d_lo) > thr
    for _ in range(60):
        mid = (d_lo + d_hi) / 2
        above = iou_at(mid) > thr
        d_lo, d_hi = np.where(above, mid, d_lo), np.where(above, d_hi, mid)
    pa, pb0, d = pa[ok], pb0[ok], d_lo[ok]
    cxb = (pb0[:, 0].astype(F64) + d).astype(F32)
    k = np.arange(-span, span + 1)
    ulp = np.spacing(np.abs(cxb)).astype(F64)
    pb = np.repeat(pb0, len(k), 0)
    pb[:, 0] = (np.repeat(cxb.astype(F64), len(k)) + np.tile(k, len(cxb)) * np.repeat(ulp, len(k))).astype(F32)
    return np.repeat(pa, len(k), 0), pb
