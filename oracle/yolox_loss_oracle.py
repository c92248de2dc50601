"""Torch restatement of the YOLOX training loss: ``YOLOXHead.get_losses`` (det/yolox/models/yolo_head.py:256-426) with
SimOTA (``get_assignments`` :436-526, ``get_in_boxes_info`` :528-595, ``dynamic_k_matching`` :597-627) and ``IOUloss``
(det/yolox/models/losses.py).

One image at a time, in the reference's op sequence, on any device and in the dtype of ``outputs`` (fp64 on the CPU for
the tests, fp32 on CUDA as the benchmark's baseline).  Where torch leaves an order open the rules of DESIGN.md §7q are
used: the k cheapest anchors of a GT are taken by a stable sort (equal cost: lower anchor index first), and an anchor
chosen by several GTs goes to the first minimum of its cost column over all GTs.

The ``replay_*`` functions take one stage's input as csrc/yolox_loss.cu left it in its workspace and give what that
stage must produce, so that each kernel stage can be checked on its own input.
"""
import numpy as np
import torch
import torch.nn.functional as F

CENTER_RADIUS = 2.5
REG_WEIGHT = 5.0
STRIDES = (8, 16, 32)
F32 = np.float32


# ------------------------------------------------------------------------------------------------- inputs
# The cases of tests/golden/ref_yolox_loss.npz (tools/make_golden_ref_yolox_loss.py):
# name -> (seed, B, side, C, GTs per image, kind, use_l1)
GOLDEN_CASES = {
    "s640": (1, 4, 640, 30, (0, 1, 20, 120), "plain", True),
    "s640_nol1": (2, 4, 640, 30, (0, 1, 20, 120), "plain", False),
    "s448": (3, 2, 448, 30, (8, 30), "plain", True),
    "s832": (4, 2, 832, 30, (30, 8), "plain", False),
    "tiny": (5, 2, 640, 30, (10, 25), "tiny", True),
    "border": (6, 2, 640, 30, (12, 20), "border", True),
    "dup": (7, 2, 640, 30, (10, 21), "dup", True),
}
# the upstream weights of the golden gradients: each term's gradient is told apart from the others
LOSS_WEIGHTS = {"loss_iou": 1.0, "loss_conf": 0.5, "loss_cls": 2.0, "loss_l1": 0.25}


def anchor_grid(side, strides=STRIDES, dtype=torch.float32, device="cpu"):
    """(x_shifts, y_shifts, expanded_strides) as YOLOXHead.forward hands them to get_losses: one [1, h*w] tensor per
    level, grid cells in row-major order."""
    xs, ys, es = [], [], []
    for s in strides:
        n = side // s
        yv, xv = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
        xs.append(xv.reshape(1, -1).to(dtype=dtype, device=device))
        ys.append(yv.reshape(1, -1).to(dtype=dtype, device=device))
        es.append(torch.full((1, n * n), float(s), dtype=dtype, device=device))
    return xs, ys, es


def decode(raw, x_shifts, y_shifts, expanded_strides):
    """The head's training decode (get_output_and_grid): raw [B, A, 5+C] -> outputs with (xy + grid) * stride and
    exp(wh) * stride; objectness and class logits unchanged.  Differentiable."""
    gx = torch.cat(x_shifts, 1)[..., None]
    gy = torch.cat(y_shifts, 1)[..., None]
    st = torch.cat(expanded_strides, 1)[..., None]
    return torch.cat([(raw[..., 0:1] + gx) * st, (raw[..., 1:2] + gy) * st, torch.exp(raw[..., 2:4]) * st, raw[..., 4:]],
                     -1)


def make_labels(g, B, side, C, n_gts, kind="plain", M=120):
    """labels [B, M, 5] fp32 = (class, cx, cy, w, h), the first n_gts[b] rows of image b filled.
    kind: plain | tiny (1..5 px boxes, candidates only through the centre region) | border (centres on the image
    border) | dup (every GT twice, adjacent: exact cost ties and conflicts) | nocand (boxes far right of the image: no
    candidate anchor at all)."""
    lab = torch.zeros(B, M, 5, dtype=torch.float64)
    for b, n in enumerate(n_gts):
        if n == 0:
            continue
        m = (n + 1) // 2 if kind == "dup" else n
        cls = torch.randint(0, C, (m,), generator=g).double()
        c = torch.rand(m, 2, generator=g, dtype=torch.float64) * side
        wh = 12 + torch.rand(m, 2, generator=g, dtype=torch.float64) * (0.45 * side - 12)
        if kind == "tiny":
            wh = 1 + torch.rand(m, 2, generator=g, dtype=torch.float64) * 4
        elif kind == "border":
            edge = torch.randint(0, 2, (m, 2), generator=g).double() * side
            pick = torch.randint(0, 2, (m,), generator=g)
            c[torch.arange(m), pick] = edge[torch.arange(m), pick] + (torch.rand(m, generator=g, dtype=torch.float64)
                                                                       - 0.5) * 8
        elif kind == "nocand":
            c[:, 0] = side + 400 + c[:, 0]
            wh = 12 + torch.rand(m, 2, generator=g, dtype=torch.float64) * 60
        rows = torch.cat([cls[:, None], c, wh], 1)
        if kind == "dup":
            rows = rows.repeat_interleave(2, 0)[:n]
        lab[b, :n] = rows
    return lab.float()


def make_case(seed, B, side, C, n_gts, kind="plain", M=120):
    """Seeded inputs of get_losses: (x_shifts, y_shifts, expanded_strides, labels, raw) in fp32 on the CPU, raw
    [B, A, 5+C] the head's raw output (decode() gives ``outputs``, raw[..., :4] is ``origin_preds``)."""
    g = torch.Generator().manual_seed(seed)
    xs, ys, es = anchor_grid(side)
    A = sum(x.shape[1] for x in xs)
    raw = torch.randn(B, A, 5 + C, generator=g, dtype=torch.float64)
    raw[..., :2] *= 0.6
    raw[..., 2:4] = raw[..., 2:4] * 0.6 + 1.1
    raw[..., 4:] = raw[..., 4:] * 1.5 - 2.0
    labels = make_labels(g, B, side, C, n_gts, kind, M)
    return xs, ys, es, labels, raw.float()


# ------------------------------------------------------------------------------------------------- assignment
def in_boxes_info(gt, xs, ys, st):
    """gt [G, 4] (cx, cy, w, h); xs, ys, st [A] -> (candidate [A], in_box [G, A], in_centre [G, A]).  Strict > 0 on the
    four deltas against the box and against c +- 2.5 stride (get_in_boxes_info)."""
    xc = (xs * st + 0.5 * st)[None]
    yc = (ys * st + 0.5 * st)[None]
    cx, cy, w, h = (gt[:, i:i + 1] for i in range(4))
    box = torch.stack([xc - (cx - 0.5 * w), yc - (cy - 0.5 * h), (cx + 0.5 * w) - xc, (cy + 0.5 * h) - yc], 2)
    r = CENTER_RADIUS * st[None]
    ctr = torch.stack([xc - (cx - r), yc - (cy - r), (cx + r) - xc, (cy + r) - yc], 2)
    in_box = box.min(2).values > 0
    in_ctr = ctr.min(2).values > 0
    return in_box.any(0) | in_ctr.any(0), in_box, in_ctr


def pair_iou(a, b):
    """bboxes_iou(a, b, xyxy=False): [Ga, Gb], no epsilon."""
    tl = torch.max(a[:, None, :2] - a[:, None, 2:] / 2, b[None, :, :2] - b[None, :, 2:] / 2)
    br = torch.min(a[:, None, :2] + a[:, None, 2:] / 2, b[None, :, :2] + b[None, :, 2:] / 2)
    inter = (br - tl).prod(2) * (tl < br).to(tl.dtype).prod(2)
    return inter / (a[:, 2:].prod(1)[:, None] + b[:, 2:].prod(1)[None] - inter)


def dynamic_ks(ious):
    """ious [G, n_cand] -> k per GT: max(1, int(sum of the min(10, n_cand) largest IoUs))."""
    top = torch.topk(ious, min(10, ious.shape[1]), dim=1).values
    return top.sum(1).int().clamp(min=1).tolist()


def choose(cost, ks):
    """Per GT the k cheapest columns (stable: equal cost -> lower column); columns taken by several GTs go to the
    first minimum of the column over all GTs.  -> (matching [G, n] uint8)."""
    m = torch.zeros_like(cost, dtype=torch.uint8)
    for g, k in enumerate(ks):
        m[g, torch.sort(cost[g], stable=True).indices[:k]] = 1
    multi = m.sum(0) > 1
    if bool(multi.any()):
        arg = cost[:, multi].min(0).indices
        m[:, multi] = 0
        m[arg, multi.nonzero()[:, 0]] = 1
    return m


def pair_costs(gt, gt_cls, boxes, obj, cls, num_classes):
    """GT x anchor IoU and unpenalised cost: BCE of sqrt(sigmoid(cls) * sigmoid(obj)) against the one-hot class, summed,
    plus 3 * -log(iou + 1e-8).  boxes [n, 4], obj [n, 1], cls [n, C] -> (ious [G, n], cost0 [G, n])."""
    G, n = gt.shape[0], boxes.shape[0]
    ious = pair_iou(gt, boxes)
    onehot = F.one_hot(gt_cls.to(torch.int64), num_classes).to(boxes.dtype)
    p = (cls.sigmoid() * obj.sigmoid()).sqrt()
    cls_cost = F.binary_cross_entropy(p[None].expand(G, n, num_classes), onehot[:, None].expand(G, n, num_classes),
                                      reduction="none").sum(-1)
    return ious, cls_cost + 3.0 * -torch.log(ious + 1e-8)


@torch.no_grad()
def assign_image(gt, gt_cls, boxes, obj, cls, xs, ys, st, num_classes):
    """One image's SimOTA.  -> dict with cand [A] bool, ious / cost [G, n_cand], ks, fg [A] bool, matched [A] long
    (-1 off fg), iou_t [A] (IoU with the matched GT)."""
    A, G = boxes.shape[0], gt.shape[0]
    cand, in_box, in_ctr = in_boxes_info(gt, xs, ys, st)
    out = dict(cand=cand, fg=torch.zeros(A, dtype=torch.bool, device=boxes.device),
               matched=torch.full((A,), -1, dtype=torch.long, device=boxes.device),
               iou_t=torch.zeros(A, dtype=boxes.dtype, device=boxes.device), ks=[0] * G)
    n = int(cand.sum())
    if n == 0:   # no candidate anchor: the GTs take nothing (the reference fails here)
        return out
    both = (in_box & in_ctr)[:, cand]
    ious, cost0 = pair_costs(gt, gt_cls, boxes[cand], obj[cand], cls[cand], num_classes)
    cost = cost0 + 100000.0 * (~both)
    ks = dynamic_ks(ious)
    m = choose(cost, ks)
    fg_c = m.sum(0) > 0
    idx = cand.nonzero()[:, 0][fg_c]
    out["fg"][idx] = True
    out["matched"][idx] = m[:, fg_c].argmax(0)
    out["iou_t"][idx] = (m.to(ious.dtype) * ious).sum(0)[fg_c]
    out.update(ious=ious, cost0=cost0, cost=cost, ks=ks)
    return out


# ------------------------------------------------------------------------------------------------- losses
def iou_loss(pred, target):
    """IOUloss(loss_type="iou"): 1 - iou^2, +1e-16 in the denominator."""
    tl = torch.max(pred[:, :2] - pred[:, 2:] / 2, target[:, :2] - target[:, 2:] / 2)
    br = torch.min(pred[:, :2] + pred[:, 2:] / 2, target[:, :2] + target[:, 2:] / 2)
    en = (tl < br).to(tl.dtype).prod(1)
    inter = torch.prod(br - tl, 1) * en
    union = torch.prod(pred[:, 2:], 1) + torch.prod(target[:, 2:], 1) - inter
    return 1 - (inter / (union + 1e-16)) ** 2


def losses_from_assignment(outputs, origin_preds, labels, fg, matched, iou_t, xs, ys, st, num_classes, use_l1):
    """The four loss terms given an assignment (fg [B, A] bool, matched [B, A] long, iou_t [B, A]), differentiable in
    outputs / origin_preds.  -> (loss_iou * 5, loss_obj, loss_cls, loss_l1, num_fg)."""
    B, A = fg.shape
    rows = fg.reshape(-1)
    bi = torch.arange(B, device=fg.device)[:, None].expand(B, A).reshape(-1)[rows]
    gi = matched.reshape(-1)[rows]
    gt = labels[bi, gi, 1:5].to(outputs.dtype)
    cls_t = F.one_hot(labels[bi, gi, 0].to(torch.int64), num_classes).to(outputs.dtype) * iou_t.reshape(-1)[rows, None]
    num_fg = max(int(rows.sum()), 1)
    li = iou_loss(outputs[..., :4].reshape(-1, 4)[rows], gt).sum() / num_fg
    lo = F.binary_cross_entropy_with_logits(outputs[..., 4].reshape(-1), fg.reshape(-1).to(outputs.dtype),
                                            reduction="none").sum() / num_fg
    lc = F.binary_cross_entropy_with_logits(outputs[..., 5:].reshape(-1, num_classes)[rows], cls_t,
                                            reduction="none").sum() / num_fg
    ll = 0.0
    if use_l1:
        a = torch.arange(A, device=fg.device)[None].expand(B, A).reshape(-1)[rows]
        s = st[a]
        tgt = torch.stack([gt[:, 0] / s - xs[a], gt[:, 1] / s - ys[a], torch.log(gt[:, 2] / s + 1e-8),
                           torch.log(gt[:, 3] / s + 1e-8)], 1)
        ll = (origin_preds.reshape(-1, 4)[rows] - tgt).abs().sum() / num_fg
    return REG_WEIGHT * li, lo, lc, ll, num_fg


def num_labels(labels):
    """GTs per image: rows with a positive sum, counted; they are taken as the first rows (even past a zero row)."""
    return (labels.sum(2) > 0).sum(1).tolist()


def get_losses(head, imgs, x_shifts, y_shifts, expanded_strides, labels, outputs, origin_preds, dtype,
               empty_cache=False, trace=None):
    """Reference signature.  Computes in outputs.dtype; ``empty_cache`` repeats the reference's per-image
    torch.cuda.empty_cache(); ``trace`` (a list) receives each image's assign_image dict."""
    C = head.num_classes
    xs = torch.cat(x_shifts, 1)[0].to(outputs.dtype)
    ys = torch.cat(y_shifts, 1)[0].to(outputs.dtype)
    st = torch.cat(expanded_strides, 1)[0].to(outputs.dtype)
    B, A = outputs.shape[:2]
    fg = torch.zeros(B, A, dtype=torch.bool, device=outputs.device)
    matched = torch.zeros(B, A, dtype=torch.long, device=outputs.device)
    iou_t = torch.zeros(B, A, dtype=outputs.dtype, device=outputs.device)
    nl = num_labels(labels)
    for b in range(B):
        G = nl[b]
        if G == 0:
            if trace is not None:
                trace.append(None)
            continue
        gt = labels[b, :G, 1:5].to(outputs.dtype)
        o = outputs[b].detach()
        r = assign_image(gt, labels[b, :G, 0], o[:, :4], o[:, 4:5], o[:, 5:], xs, ys, st, C)
        fg[b], matched[b], iou_t[b] = r["fg"], r["matched"].clamp(min=0), r["iou_t"]
        if trace is not None:
            trace.append(r)
        if empty_cache:
            torch.cuda.empty_cache()
    li, lo, lc, ll, num_fg = losses_from_assignment(outputs, torch.cat(origin_preds, 1) if head.use_l1 else None,
                                                    labels, fg, matched, iou_t, xs, ys, st, C, head.use_l1)
    return ({"num_fg": num_fg / max(sum(nl), 1)},
            {"loss_iou": li, "loss_conf": lo, "loss_l1": ll, "loss_cls": lc})


# ------------------------------------------------------------------------------------------------- stage replays
def replay_candidates(gt, xs, ys, st):
    """fp32 NumPy replica of the candidate test, one rounding per operation.  gt [G, 4], xs / ys / st [A] float32 ->
    (cand [A] bool, in_both [G, A] bool)."""
    gt, xs, ys, st = (np.asarray(v, F32) for v in (gt, xs, ys, st))
    half, rad = F32(0.5), F32(CENTER_RADIUS)
    xc = (xs * st + half * st)[None]
    yc = (ys * st + half * st)[None]
    cx, cy, w, h = (gt[:, i:i + 1] for i in range(4))
    box = np.stack([xc - (cx - half * w), yc - (cy - half * h), (cx + half * w) - xc, (cy + half * h) - yc]).min(0) > 0
    r = rad * st[None]
    ctr = np.stack([xc - (cx - r), yc - (cy - r), (cx + r) - xc, (cy + r) - yc]).min(0) > 0
    return box.any(0) | ctr.any(0), box & ctr


def replay_k(iou_rows):
    """iou_rows [G, n_cand] (the kernel's IoUs over the image's candidates) -> (k [G], fp64 top-10 sums [G])."""
    iou_rows = np.asarray(iou_rows, np.float64)
    top = -np.sort(-iou_rows, axis=1)[:, :min(10, iou_rows.shape[1])]
    s = top.sum(1)
    return np.maximum(1, s.astype(np.int64)), s


def replay_choice(cost, ks):
    """cost [G, n_cand] (the kernel's fp32 costs), ks [G] -> (chosen: list of per-GT column arrays, fg [n_cand] bool,
    matched [n_cand] int, -1 off fg), by the tie rules of ``choose``."""
    cost = torch.as_tensor(np.asarray(cost, F32))
    chosen = [np.sort(torch.sort(cost[g], stable=True).indices[:int(k)].numpy()) for g, k in enumerate(ks)]
    m = choose(cost, [int(k) for k in ks]).numpy()
    fg = m.sum(0) > 0
    return chosen, fg, np.where(fg, m.argmax(0), -1)
