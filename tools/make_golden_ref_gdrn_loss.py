"""Generate tests/golden/ref_gdrn_loss.npz by running the REFERENCE's own ``GDRN_DoubleMask.gdrn_loss``
(core/gdrn_modeling/models/GDRN_double_mask.py, called unbound with a stub ``self`` that holds the USE_MTL log
variances) with its ``PyPMLoss`` and ``get_closest_rot_batch``, imported read-only from the checkout that
GDRN_REFERENCE_SRC names with the import stubs of make_golden_ref_heads.py, on the CPU in fp32.

Inputs are not stored: ``oracle.gdrn_loss_oracle.make_case`` regenerates them from each case's seed.  Stored per case
(keys prefixed ``<case>/``): the losses in LOSS_WEIGHTS order (NaN where the config has no such term), the chosen
symmetry index per ROI (-1 = R_gt itself) and the gap between the best and second-best ``re`` of distinct candidates in
degrees (inf without a symmetry), the autograd gradients of sum(LOSS_WEIGHTS[k] * loss_k) for out_rot, out_centroid and
out_trans_z in full, and for every dense map its sum and its values at the seeded positions of
``oracle.gdrn_loss_oracle.sample_positions``.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_ref_gdrn_loss.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
sys.path.insert(0, ROOT)

from oracle import gdrn_loss_oracle as O  # noqa: E402


def recording_closest(orig, re, record):
    """get_closest_rot_batch as the reference runs it, recording per ROI the chosen index and the decision gap with the
    reference's own ``re``."""

    def fn(pred_rots, gt_rots, sym_infos):
        idx, gap = [], []
        for i in range(pred_rots.shape[0]):
            S = sym_infos[i]
            if S is None:
                idx.append(-1)
                gap.append(np.inf)
                continue
            pe, rg = pred_rots[i].detach().cpu().numpy(), gt_rots[i].cpu().numpy()
            cands = [rg] + [rg.dot(S[k]) for k in range(S.shape[0])]
            errs = [re(pe, c) for c in cands]
            best, bi = errs[0], -1
            for k in range(S.shape[0]):
                if errs[k + 1] < best:
                    best, bi = errs[k + 1], k
            others = [e for c, e in zip(cands, errs) if not np.array_equal(c, cands[bi + 1])]
            idx.append(bi)
            gap.append(float(min(others) - best) if others else np.inf)
        record["sym_idx"], record["sym_gap"] = np.array(idx, np.int32), np.array(gap, np.float64)
        return orig(pred_rots, gt_rots, sym_infos)

    return fn


def run_reference(gdrn_loss, name):
    case, cfg_kw = O.GOLDEN_CASES[name]
    d = O.to(O.make_case(**case), torch.float32)
    cfg = O.make_cfg(**cfg_kw)
    model = O.MtlModel(torch.float32)
    args = {k: d[k] for k in ("out_mask_vis", "out_mask_full", "gt_mask_trunc", "gt_mask_visib", "gt_mask_obj",
                              "gt_mask_full", "out_x", "out_y", "out_z", "gt_xyz", "gt_xyz_bin", "out_region",
                              "gt_region", "out_rot", "gt_rot", "out_trans", "gt_trans", "out_centroid", "out_trans_z",
                              "gt_trans_ratio", "gt_points", "sym_infos", "extents")}
    losses = gdrn_loss(model, cfg, **args)
    O.weighted_total(losses).backward()
    rec = {"losses": np.array([float(losses[k].detach()) if k in losses else np.nan for k in O.LOSS_WEIGHTS])}
    for k in O.SMALL:
        g = d[k].grad
        rec["grad_" + k] = np.zeros(d[k].shape, np.float32) if g is None else g.numpy()
    for k in O.DENSE:
        g = d[k].grad
        g = np.zeros(d[k].shape, np.float32) if g is None else g.numpy()
        rec["gsum_" + k] = np.float64(g.astype(np.float64).sum())
        rec["gsamp_" + k] = g.reshape(-1)[O.sample_positions(k, g.shape)]
    return rec


def main():
    assert REF and os.path.isdir(REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_ref_heads as mh

    mh.STUB_TOPLEVEL.update({"torchvision"})
    sys.meta_path.insert(0, mh.StubFinder())
    for _n, _v in (("float", float), ("int", int), ("bool", bool), ("maximum_sctype", lambda t: np.float64)):
        if not hasattr(np, _n):   # NumPy 2 removed these; the reference's modules use them at import time
            setattr(np, _n, _v)
    sys.path.insert(0, REF)
    from core.gdrn_modeling.losses import pm_loss
    from core.gdrn_modeling.models.GDRN_double_mask import GDRN_DoubleMask
    from lib.pysixd.pose_error import re

    data = {}
    orig = pm_loss.get_closest_rot_batch
    for name in O.GOLDEN_CASES:
        record = {}
        pm_loss.get_closest_rot_batch = recording_closest(orig, re, record)
        try:
            rec = run_reference(GDRN_DoubleMask.gdrn_loss, name)
        finally:
            pm_loss.get_closest_rot_batch = orig
        B = O.GOLDEN_CASES[name][0]["B"]
        rec["sym_idx"] = record.get("sym_idx", np.full(B, -1, np.int32))
        rec["sym_gap"] = record.get("sym_gap", np.full(B, np.inf))
        for k, v in rec.items():
            data[f"{name}/{k}"] = v
        print(name, "losses", rec["losses"], "min gap", rec["sym_gap"].min())
    path = os.path.join(ROOT, "tests", "golden", "ref_gdrn_loss.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
