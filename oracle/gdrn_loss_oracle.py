"""Torch restatement of the GDRN training loss: ``GDRN_DoubleMask.gdrn_loss``
(core/gdrn_modeling/models/GDRN_double_mask.py:287-536) with ``PyPMLoss`` (core/gdrn_modeling/losses/pm_loss.py, R only)
and ``get_closest_rot_batch`` / ``get_closest_rot`` / ``pose_error.re`` (core/utils/pose_utils.py:472-528,
lib/pysixd/pose_error.py).

The reference's op sequence, on any device and in the dtype of the inputs (fp64 on the CPU for the tests, fp32 on CUDA
as the benchmark's baseline, where the closest rotation is chosen by the same per-ROI host loop as the reference's).

The ``replay_*`` functions take one stage's input as csrc/gdrn_loss.cu left it in its workspace and give what that stage
must produce, so that each kernel stage can be checked on its own input.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from gdrnpp_bop2022_b200.bop_eval import get_symmetry_transformations

TILE = 512   # pixels per CTA of the dense kernels


class Node(dict):
    """A config node with attribute access and ``.get``, as the reference's mmcv Config gives."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __setattr__(self, k, v):
        self[k] = v


def make_cfg(freeze=False, use_mtl=False, z_type="REL", **loss):
    """cfg.MODEL.POSE_NET with configs/_base_/gdrn_base.py's LOSS_CFG, overridden by ``loss``; PM_LOSS_SYM on and the
    full-mask term at weight 1, as the shipped configs set them."""
    lc = Node(XYZ_LOSS_TYPE="L1", XYZ_LOSS_MASK_GT="visib", XYZ_LW=1.0, FULL_MASK_LOSS_TYPE="L1", FULL_MASK_LW=1.0,
              MASK_LOSS_TYPE="L1", MASK_LOSS_GT="trunc", MASK_LW=1.0, REGION_LOSS_TYPE="CE", REGION_LOSS_MASK_GT="visib",
              REGION_LW=1.0, NUM_PM_POINTS=3000, PM_LOSS_TYPE="L1", PM_SMOOTH_L1_BETA=1.0, PM_LOSS_SYM=True,
              PM_NORM_BY_EXTENT=False, PM_R_ONLY=True, PM_DISENTANGLE_T=False, PM_DISENTANGLE_Z=False,
              PM_T_USE_POINTS=True, PM_LW=1.0, ROT_LOSS_TYPE="angular", ROT_LW=0.0, CENTROID_LOSS_TYPE="L1",
              CENTROID_LW=1.0, Z_LOSS_TYPE="L1", Z_LW=1.0, TRANS_LOSS_TYPE="L1", TRANS_LOSS_DISENTANGLE=True, TRANS_LW=0.0,
              BIND_LOSS_TYPE="L1", BIND_LW=0.0)
    lc.update(loss)
    net = Node(GEO_HEAD=Node(FREEZE=freeze), PNP_NET=Node(TRANS_TYPE="centroid_z", Z_TYPE=z_type), LOSS_CFG=lc,
               USE_MTL=use_mtl)
    return Node(MODEL=Node(POSE_NET=net))


# ------------------------------------------------------------------------------------------------- inputs
def sym_tables():
    """The symmetry kinds of the cases: 'two' (the identity and a discrete half turn about z, as
    get_symmetry_transformations gives a box-like object) and 'cont' (a continuous symmetry about z with a discrete
    flip about x, discretised at max_sym_disc_step = 0.01: 2 x 314 rotations), both f32 [K,3,3] as the batcher holds."""
    two = get_symmetry_transformations({"symmetries_discrete": [np.diag([-1.0, -1.0, 1.0, 1.0])]}, 0.01)
    flip = np.diag([1.0, -1.0, -1.0, 1.0])
    cont = get_symmetry_transformations({"symmetries_discrete": [flip],
                                         "symmetries_continuous": [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]}, 0.01)
    return {k: np.array([s["R"] for s in v], np.float32) for k, v in (("two", two), ("cont", cont))}


def _random_rot(rng):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _axis_angle(rng, deg):
    ax = rng.standard_normal(3)
    ax /= np.linalg.norm(ax)
    a = math.radians(deg)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + math.sin(a) * K + (1 - math.cos(a)) * K @ K


def make_case(seed, B, syms=("none",), R=64, N=300, H=64, W=64, empty_visib=(), all_empty=False, tables=None):
    """Seeded inputs of one call, fp32 on the CPU: a dict of the reference method's tensor arguments plus sym_infos (the
    same array object for every ROI of one kind, as the batcher hands them out).  ROI b takes symmetry kind
    syms[b % len(syms)] ('none', 'two' or 'cont'); its predicted rotation is a GT-equivalent rotation 2-20 degrees off,
    so that the closest symmetric GT is not R_gt itself.  ROIs in ``empty_visib`` have an all-zero visible mask;
    ``all_empty`` zeroes every GT mask."""
    rng = np.random.default_rng(seed)
    tables = tables or sym_tables()
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))  # noqa: E731
    blobs = rng.random((4, B, H, W))
    obj = blobs[0] > 0.35
    visib = obj & (blobs[1] > 0.3)
    trunc = visib & (blobs[2] > 0.1)
    full = obj | (blobs[3] > 0.8)
    for b in empty_visib:
        visib[b] = trunc[b] = False
    if all_empty:
        obj[:] = visib[:] = trunc[:] = full[:] = False
    sym_infos, gt_rot, out_rot = [], [], []
    for b in range(B):
        kind = syms[b % len(syms)]
        S = None if kind == "none" else tables[kind]
        sym_infos.append(S)
        Rg = _random_rot(rng)
        Rs = Rg if S is None else Rg @ S[rng.integers(S.shape[0])].astype(np.float64)
        gt_rot.append(Rg)
        out_rot.append(Rs @ _axis_angle(rng, rng.uniform(2, 20)))
    ext = rng.uniform(0.05, 0.3, (B, 3))
    pts = (rng.random((B, N, 3)) - 0.5) * ext[:, None, :]
    d = {
        "out_mask_vis": f(rng.standard_normal((B, 1, H, W)) * 2), "out_mask_full": f(rng.standard_normal((B, 1, H, W)) * 2),
        "gt_mask_trunc": f(trunc), "gt_mask_visib": f(visib), "gt_mask_obj": f(obj), "gt_mask_full": f(full),
        "out_x": f(rng.random((B, 1, H, W))), "out_y": f(rng.random((B, 1, H, W))), "out_z": f(rng.random((B, 1, H, W))),
        "gt_xyz": f(rng.random((B, 3, H, W))), "gt_xyz_bin": None,
        "out_region": f(rng.standard_normal((B, R + 1, H, W)) * 3), "gt_region": torch.from_numpy(
            rng.integers(0, R + 1, (B, H, W))).to(torch.int64),
        "out_rot": f(np.stack(out_rot)), "gt_rot": f(np.stack(gt_rot)), "out_trans": None,
        "gt_trans": f(np.c_[rng.uniform(-0.2, 0.2, (B, 2)), rng.uniform(0.5, 1.5, B)]),
        "out_centroid": f(rng.standard_normal((B, 2)) * 0.1), "out_trans_z": f(rng.uniform(0.5, 1.5, B)),
        "gt_trans_ratio": f(np.c_[rng.standard_normal((B, 2)) * 0.1, rng.uniform(0.5, 1.5, B)]),
        "gt_points": f(pts), "sym_infos": sym_infos, "extents": f(ext),
    }
    return d


# The cases of tests/golden/ref_gdrn_loss.npz (tools/make_golden_ref_gdrn_loss.py):
# name -> (make_case kwargs, make_cfg kwargs)
GOLDEN_CASES = {
    "b1": (dict(seed=1, B=1, syms=("none",)), dict(PM_NORM_BY_EXTENT=True)),
    "b8_two_bce": (dict(seed=2, B=8, syms=("two", "none")),
                   dict(MASK_LOSS_TYPE="BCE", FULL_MASK_LOSS_TYPE="BCE", z_type="ABS")),
    "b48_mixed": (dict(seed=3, B=48, syms=("cont", "none", "two"), empty_visib=(5,)), dict(PM_NORM_BY_EXTENT=True)),
    "b36_cont_mtl": (dict(seed=4, B=36, syms=("cont",)), dict(use_mtl=True, XYZ_LOSS_MASK_GT="obj",
                                                                 REGION_LOSS_MASK_GT="trunc", MASK_LOSS_GT="full")),
    "b4_freeze": (dict(seed=5, B=4, syms=("two",)), dict(freeze=True)),
    "b3_empty": (dict(seed=6, B=3, syms=("none", "two"), all_empty=True), dict(PM_LOSS_SYM=False, FULL_MASK_LW=0.0)),
}
# the upstream weights of the golden gradients: each term's gradient is told apart from the others
LOSS_WEIGHTS = {"loss_coor_x": 1.0, "loss_coor_y": 0.5, "loss_coor_z": 2.0, "loss_mask": 0.75, "loss_mask_full": 1.5,
                "loss_region": 0.25, "loss_PM_R": 3.0, "loss_centroid": 0.6, "loss_z": 1.25}
DENSE = ("out_x", "out_y", "out_z", "out_mask_vis", "out_mask_full", "out_region")
SMALL = ("out_rot", "out_centroid", "out_trans_z")
N_SAMPLES = 64


class MtlModel:
    """A model stand-in holding the USE_MTL log variances, one per loss key, as the reference's model does."""

    def __init__(self, dtype=torch.float64, device="cpu"):
        for i, k in enumerate(LOSS_WEIGHTS):
            setattr(self, k.replace("loss_", "log_var_"),
                    torch.tensor(0.1 * (i - 4), dtype=dtype, device=device, requires_grad=True))


def sample_positions(name, shape):
    """The seeded flat positions of a dense gradient stored in the golden file."""
    rng = np.random.default_rng([len(name), *map(ord, name)])
    return rng.integers(0, int(np.prod(shape)), N_SAMPLES)


# ------------------------------------------------------------------------------------------------- the loss
def re_deg(R_est, R_gt):
    """pose_error.re in the arrays' dtype."""
    tr = np.trace(R_est.dot(R_gt.T))
    tr = tr if tr <= 3 else 3
    return np.rad2deg(np.arccos(min(1.0, max(-1.0, 0.5 * (tr - 1.0)))))


def closest_rot_batch(pred_rots, gt_rots, sym_infos):
    """get_closest_rot_batch: one host round trip per ROI, as the reference.  -> (closest [B,3,3] like gt_rots, chosen
    index per ROI (-1 = R_gt itself, k = R_gt S_k), gap between the best and second-best error in degrees (inf when
    there is one candidate))."""
    out = gt_rots.clone().cpu().numpy()
    idx = np.full(len(out), -1, np.int64)
    gap = np.full(len(out), np.inf)
    for i in range(len(out)):
        S = sym_infos[i]
        if S is None:
            continue
        if torch.is_tensor(S):
            S = S.cpu().numpy()
        S = S.reshape(-1, 3, 3)
        re_ = pred_rots[i].detach().cpu().numpy()
        rg = gt_rots[i].cpu().numpy()
        cands = [rg] + [rg.dot(S[k].astype(rg.dtype)) for k in range(S.shape[0])]
        errs = [re_deg(re_, c) for c in cands]
        best, bi = errs[0], -1
        for k in range(S.shape[0]):
            if errs[k + 1] < best:
                best, bi, out[i] = errs[k + 1], k, cands[k + 1]
        idx[i] = bi
        # candidates equal to the chosen rotation (an identity in the table) tie exactly and are not a margin
        others = [e for c, e in zip(cands, errs) if not np.array_equal(c, cands[bi + 1])]
        gap[i] = min(others) - best if others else np.inf
    return torch.tensor(out, device=gt_rots.device, dtype=gt_rots.dtype), idx, gap


def gdrn_loss(cfg, d, model=None, record=None):
    """The reference's gdrn_loss for the supported options; ``d`` as make_case gives it (any dtype and device).
    ``record`` (a dict or None) receives the closest-rotation index and gap."""
    net_cfg = cfg.MODEL.POSE_NET
    loss_cfg = net_cfg.LOSS_CFG
    loss_dict = {}
    gt_masks = {"trunc": d["gt_mask_trunc"], "visib": d["gt_mask_visib"], "obj": d["gt_mask_obj"],
                "full": d["gt_mask_full"]}
    if not net_cfg.GEO_HEAD.FREEZE:
        m = gt_masks[loss_cfg.XYZ_LOSS_MASK_GT]
        l1 = nn.L1Loss(reduction="sum")
        for c, k in enumerate(("x", "y", "z")):
            loss_dict["loss_coor_" + k] = l1(d["out_" + k] * m[:, None], d["gt_xyz"][:, c:c + 1] * m[:, None]) / \
                m.sum().float().clamp(min=1.0) * loss_cfg.XYZ_LW
        gm = gt_masks[loss_cfg.MASK_LOSS_GT]
        fn = nn.L1Loss(reduction="mean") if loss_cfg.MASK_LOSS_TYPE == "L1" else nn.BCEWithLogitsLoss(reduction="mean")
        loss_dict["loss_mask"] = fn(d["out_mask_vis"][:, 0], gm) * loss_cfg.MASK_LW
        if loss_cfg.FULL_MASK_LW > 0:
            fn = nn.L1Loss(reduction="mean") if loss_cfg.FULL_MASK_LOSS_TYPE == "L1" else \
                nn.BCEWithLogitsLoss(reduction="mean")
            loss_dict["loss_mask_full"] = fn(d["out_mask_full"][:, 0], d["gt_mask_full"]) * loss_cfg.FULL_MASK_LW
        mr = gt_masks[loss_cfg.REGION_LOSS_MASK_GT]
        loss_dict["loss_region"] = nn.CrossEntropyLoss(reduction="sum")(
            d["out_region"] * mr[:, None], d["gt_region"].long() * mr.long()) / mr.sum().float().clamp(min=1.0) * \
            loss_cfg.REGION_LW
    if loss_cfg.PM_LW > 0:
        gt_rots = d["gt_rot"]
        if loss_cfg.PM_LOSS_SYM:
            gt_rots, idx, gap = closest_rot_batch(d["out_rot"], gt_rots, d["sym_infos"])
            if record is not None:
                record.update(sym_idx=idx, sym_gap=gap)
        pts = d["gt_points"]
        B, n = pts.shape[:2]
        est = (d["out_rot"].view(B, 1, 3, 3) @ pts.view(B, n, 3, 1)).squeeze(-1)
        tgt = (gt_rots.view(B, 1, 3, 3) @ pts.view(B, n, 3, 1)).squeeze(-1)
        w = (1.0 / d["extents"].max(1, keepdim=True)[0]).view(-1, 1, 1) if loss_cfg.PM_NORM_BY_EXTENT else 1
        loss_dict["loss_PM_R"] = 3 * nn.L1Loss(reduction="mean")(w * est, w * tgt) * loss_cfg.PM_LW
    if loss_cfg.CENTROID_LW > 0:
        loss_dict["loss_centroid"] = nn.L1Loss(reduction="mean")(d["out_centroid"], d["gt_trans_ratio"][:, :2]) * \
            loss_cfg.CENTROID_LW
    if loss_cfg.Z_LW > 0:
        gt_z = d["gt_trans_ratio"][:, 2] if net_cfg.PNP_NET.Z_TYPE == "REL" else d["gt_trans"][:, 2]
        loss_dict["loss_z"] = nn.L1Loss(reduction="mean")(d["out_trans_z"], gt_z) * loss_cfg.Z_LW
    if net_cfg.USE_MTL:
        for k in loss_dict:
            lv = getattr(model, k.replace("loss_", "log_var_"))
            loss_dict[k] = loss_dict[k] * torch.exp(-lv) + torch.log(1 + torch.exp(lv))
    return loss_dict


def to(d, dtype, device="cpu", grad=True):
    """make_case's dict in ``dtype`` on ``device``, the head outputs as fresh leaves (when ``grad``)."""
    out = {}
    for k, v in d.items():
        if torch.is_tensor(v):
            v = v.to(device=device, dtype=dtype if v.is_floating_point() else v.dtype)
            if grad and k in DENSE + SMALL:
                v = v.detach().requires_grad_(True)
        out[k] = v
    return out


def weighted_total(losses):
    return sum(LOSS_WEIGHTS[k] * v for k, v in losses.items())


# ------------------------------------------------------------------------------------------------- stage replays
def replay_partials(cfg, d, tiles):
    """Stage 1 in fp64 from the inputs: [B * tiles, 8] per-CTA sums (|dx|, |dy|, |dz|, mask, full mask, region CE, xyz
    count, region count), the pixels of a CTA being its 512-pixel tile of one ROI's plane."""
    lc = cfg.MODEL.POSE_NET.LOSS_CFG
    g = {k: v.double() if torch.is_tensor(v) and v.is_floating_point() else v for k, v in d.items()}
    gm = {"trunc": g["gt_mask_trunc"], "visib": g["gt_mask_visib"], "obj": g["gt_mask_obj"], "full": g["gt_mask_full"]}
    B = g["out_x"].shape[0]
    mx = gm[lc.XYZ_LOSS_MASK_GT].reshape(B, -1)
    terms = [((g["out_" + k] * mx.view_as(g["out_x"]) - g["gt_xyz"][:, c:c + 1] * mx.view_as(g["out_x"])).abs()
              ).reshape(B, -1) for c, k in enumerate("xyz")]

    def mterm(o, y, kind):
        o, y = o.reshape(B, -1), y.reshape(B, -1)
        return (o - y).abs() if kind == "L1" else o.clamp(min=0) - o * y + torch.log1p(torch.exp(-o.abs()))

    terms.append(mterm(g["out_mask_vis"], gm[lc.MASK_LOSS_GT], lc.MASK_LOSS_TYPE))
    terms.append(mterm(g["out_mask_full"], g["gt_mask_full"], lc.FULL_MASK_LOSS_TYPE) if lc.FULL_MASK_LW > 0
                 else torch.zeros_like(terms[0]))
    mr = gm[lc.REGION_LOSS_MASK_GT]
    logits = g["out_region"] * mr[:, None]
    lab = g["gt_region"].long() * mr.long()
    ce = torch.logsumexp(logits, 1) - logits.gather(1, lab[:, None])[:, 0]
    terms += [ce.reshape(B, -1), mx, mr.reshape(B, -1)]
    HW = mx.shape[1]
    pad = tiles * TILE - HW
    st = torch.stack([torch.nn.functional.pad(t, (0, pad)) for t in terms], -1)   # [B, tiles*512, 8]
    return st.view(B, tiles, TILE, 8).sum(2).reshape(B * tiles, 8)


def replay_lse(cfg, d):
    """Each pixel's region log-sum-exp in fp64 [B, HW]."""
    lc = cfg.MODEL.POSE_NET.LOSS_CFG
    gm = {"trunc": d["gt_mask_trunc"], "visib": d["gt_mask_visib"], "obj": d["gt_mask_obj"]}
    mr = gm[lc.REGION_LOSS_MASK_GT].double()
    return torch.logsumexp(d["out_region"].double() * mr[:, None], 1).reshape(mr.shape[0], -1)


def replay_closest(out_rot, gt_rot, sym_infos):
    """Stage 2's choice in fp64: (index per ROI, R_gt' [B,3,3], gap in degrees)."""
    rots, idx, gap = closest_rot_batch(out_rot.double().cpu(), gt_rot.double().cpu(), sym_infos)
    return idx, rots, gap


def replay_pm_sums(out_rot, rot_sel, points, w):
    """Stage 2's point sums in fp64 from the kernel's R_gt': (sum |w (R_est - R_gt') p| per ROI [B], the nine sums
    sign(.) w p^T [B,3,3] with the sign of the fp64 difference, and the count of differences within 1e-6 of 0)."""
    E, G, P = out_rot.double(), rot_sel.double(), points.double()
    w = w.double().view(-1, 1, 1)
    diff = w * torch.einsum("bij,bnj->bni", E, P) - w * torch.einsum("bij,bnj->bni", G, P)
    sums = torch.einsum("bni,bnj->bij", torch.sign(diff), w * P)
    return diff.abs().sum((1, 2)), sums, (diff.abs() < 1e-6).sum((1, 2))


def replay_map_grads(cfg, d, lse, norm, up):
    """Stage 4's map gradients by the kernel's fp32 formulas, from its log-sum-exp and normalisers and the upstream
    gradients ``up`` [9]: {name: gradient}."""
    lc = cfg.MODEL.POSE_NET.LOSS_CFG
    gm = {"trunc": d["gt_mask_trunc"], "visib": d["gt_mask_visib"], "obj": d["gt_mask_obj"], "full": d["gt_mask_full"]}
    B = d["out_x"].shape[0]
    sc = lambda u, w, n: (u * w) / n  # noqa: E731
    f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=up.device)  # noqa: E731
    out = {}
    m = gm[lc.XYZ_LOSS_MASK_GT][:, None]
    for c, k in enumerate("xyz"):
        s = sc(up[c], f32(lc.XYZ_LW), norm[0])
        out["out_" + k] = torch.sign(d["out_" + k] * m - d["gt_xyz"][:, c:c + 1] * m) * s * m
    for i, (o, y, kind, lw) in enumerate(((d["out_mask_vis"], gm[lc.MASK_LOSS_GT], lc.MASK_LOSS_TYPE, lc.MASK_LW),
                                          (d["out_mask_full"], gm["full"], lc.FULL_MASK_LOSS_TYPE, lc.FULL_MASK_LW))):
        if i == 1 and lc.FULL_MASK_LW <= 0:
            continue
        s = sc(up[3 + i], f32(lw), norm[2])
        y = y[:, None]
        out[("out_mask_vis", "out_mask_full")[i]] = (torch.sigmoid(o) - y if kind == "BCE" else torch.sign(o - y)) * s
    mr = gm[lc.REGION_LOSS_MASK_GT][:, None]
    s = sc(up[5], f32(lc.REGION_LW), norm[1])
    q = torch.exp(d["out_region"] * mr - lse.view(B, 1, *d["out_region"].shape[2:]))
    lab = (d["gt_region"].long() * mr[:, 0].long())[:, None]
    q = q - torch.zeros_like(q).scatter_(1, lab, 1.0)
    out["out_region"] = q * s * mr
    return out
