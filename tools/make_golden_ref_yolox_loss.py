"""Generate tests/golden/ref_yolox_loss.npz by running the REFERENCE's own ``YOLOXHead.get_losses``
(det/yolox/models/yolo_head.py, imported read-only from the checkout that GDRN_REFERENCE_SRC names, with the import stubs
of make_golden_ref_heads.py) on the CPU in fp32.

Inputs are not stored: ``oracle.yolox_loss_oracle.make_case`` regenerates them from each case's seed.  Stored per case
(keys prefixed ``<case>/``): the fg mask, matched GT and IoU target of every fg anchor, the four losses, the autograd
gradients of ``1 * loss_iou + 0.5 * loss_conf + 2 * loss_cls + 0.25 * loss_l1`` (``outputs`` at its non-zero rows
besides the dense objectness column, ``origin_preds`` at its non-zero rows), and per GT the two decision margins of the
reference's fp32 assignment: the gap between its k-th and (k+1)-th smallest cost, and the distance of its top-10 IoU
sum from the nearest integer.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_ref_yolox_loss.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
sys.path.insert(0, ROOT)

from oracle import yolox_loss_oracle as O  # noqa: E402

CASES = O.GOLDEN_CASES
LOSS_WEIGHTS = O.LOSS_WEIGHTS


def run_reference(head_cls, name):
    seed, B, side, C, n_gts, kind, use_l1 = CASES[name]
    xs, ys, es, labels, raw = O.make_case(seed, B, side, C, n_gts, kind)
    head = head_cls(C, width=0.25)
    head.use_l1 = use_l1
    margins = []
    orig = head.dynamic_k_matching

    def recording(cost, pair_wise_ious, gt_classes, num_gt, fg_mask):
        n = cost.shape[1]
        top = torch.topk(pair_wise_ious, min(10, n), dim=1).values.sum(1)
        ks = torch.clamp(top.int(), min=1)
        srt = torch.sort(cost, dim=1).values
        gap = [float(srt[g, k] - srt[g, k - 1]) if k < n else np.inf for g, k in enumerate(ks.tolist())]
        margins.append(np.stack([np.array(gap), (top - top.round()).abs().double().numpy()], 1))
        return orig(cost, pair_wise_ious, gt_classes, num_gt, fg_mask)

    head.dynamic_k_matching = recording
    raw = raw.clone().requires_grad_(True)
    outputs = O.decode(raw, xs, ys, es).detach().requires_grad_(True)
    origin = raw[..., :4].detach().clone().requires_grad_(True)
    levels = torch.split(origin, [x.shape[1] for x in xs], 1)
    out, losses = head.get_losses(None, xs, ys, es, labels, outputs, list(levels), dtype=torch.float32)
    total = sum(w * losses[k] for k, w in LOSS_WEIGHTS.items() if torch.is_tensor(losses[k]))
    total.backward()
    g_out = outputs.grad.numpy()
    g_org = origin.grad.numpy() if origin.grad is not None else np.zeros(origin.shape, np.float32)
    rec = {}
    fg = (np.abs(g_out[..., :4]).sum(-1) + np.abs(g_out[..., 5:]).sum(-1)) > 0
    rec["grad_obj"] = g_out[..., 4]
    rec["grad_rows"] = np.stack(np.nonzero(fg), 1).astype(np.int32)
    rec["grad_out_rows"] = g_out[fg]
    rows_o = np.abs(g_org).sum(-1) > 0
    rec["grad_origin_rows_idx"] = np.stack(np.nonzero(rows_o), 1).astype(np.int32)
    rec["grad_origin_rows"] = g_org[rows_o]
    rec["losses"] = np.array([float(losses[k].detach()) if torch.is_tensor(losses[k]) else losses[k] for k in ("loss_iou", "loss_conf", "loss_cls", "loss_l1")], np.float64)
    rec["margins"] = np.concatenate(margins, 0) if margins else np.zeros((0, 2))
    return rec


def assignment(head_cls, name):
    """The reference's fg / matched / IoU target, read back through its own dynamic_k_matching results."""
    seed, B, side, C, n_gts, kind, use_l1 = CASES[name]
    xs, ys, es, labels, raw = O.make_case(seed, B, side, C, n_gts, kind)
    head = head_cls(C, width=0.25)
    outputs = O.decode(raw, xs, ys, es)
    xcat, ycat, ecat = torch.cat(xs, 1), torch.cat(ys, 1), torch.cat(es, 1)
    A = outputs.shape[1]
    fg = np.zeros((B, A), bool)
    matched = np.full((B, A), -1, np.int32)
    iou_t = np.zeros((B, A), np.float32)
    nl = O.num_labels(labels)
    for b in range(B):
        if nl[b] == 0:
            continue
        gt_cls, fg_mask, ious, m_inds, _ = head.get_assignments(
            b, nl[b], A, labels[b, :nl[b], 1:5], labels[b, :nl[b], 0], outputs[b, :, :4], ecat, xcat, ycat,
            outputs[..., 5:], outputs[..., :4], outputs[..., 4:5], labels, None)
        fg[b] = fg_mask.numpy()
        matched[b, fg[b]] = m_inds.numpy()
        iou_t[b, fg[b]] = ious.numpy()
    return fg, matched, iou_t


def main():
    assert REF and os.path.isdir(REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_ref_heads as mh

    mh.STUB_TOPLEVEL.update({"torchvision"})
    sys.meta_path.insert(0, mh.StubFinder())
    sys.path.insert(0, REF)
    from det.yolox.models.yolo_head import YOLOXHead

    data = {}
    for name in CASES:
        rec = run_reference(YOLOXHead, name)
        fg, matched, iou_t = assignment(YOLOXHead, name)
        rec["fg_idx"] = np.stack(np.nonzero(fg), 1).astype(np.int32)
        rec["matched"] = matched[fg]
        rec["iou_t"] = iou_t[fg]
        for k, v in rec.items():
            data[f"{name}/{k}"] = v
        print(name, "fg", int(fg.sum()), "losses", rec["losses"], "min margins", rec["margins"].min(0)
              if len(rec["margins"]) else None)
    path = os.path.join(ROOT, "tests", "golden", "ref_yolox_loss.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
