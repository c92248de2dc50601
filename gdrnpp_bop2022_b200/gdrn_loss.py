"""GDRN training loss on the GPU (DESIGN.md §7r): ``GDRN_DoubleMask.gdrn_loss``
(core/gdrn_modeling/models/GDRN_double_mask.py:287-536) as one set of launches of libgdrn_b200.so per batch
(csrc/gdrn_loss.cu): the coordinate, mask, full-mask and region terms over the head's maps, symmetry-aware point matching
with the closest symmetric GT rotation chosen on the device, the centroid and z terms, and their gradients through
autograd.  No CPU fallback.

``gdrn_loss`` has the reference method's signature with ``self`` renamed to ``model``, so
``GDRN_DoubleMask.gdrn_loss = gdrn_loss.gdrn_loss`` swaps it into the reference's own training model.  It returns the
reference's keys for the same config, each a 0-d fp32 device tensor already times its weight.  The options it covers are
the ones every shipped config resolves to (``check_cfg``); anything else raises ``NotImplementedError`` naming the option
before any launch.

Symmetry tables are uploaded once per distinct object: ``sym_infos`` entries are looked up by ``id()`` in a registry that
keeps them alive, so a data loader that hands out the same per-object arrays every step uploads nothing in steady state.
"""
import numpy as np
import torch

from . import _lib

LAYOUT_NAMES = ("partial", "partial_err", "lse", "sym_idx", "rot_sel", "pm_abs", "pm_sign", "sym_err", "norm", "result")
RESULT_KEYS = ("loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask", "loss_mask_full", "loss_region", "loss_PM_R",
               "loss_centroid", "loss_z")
F_GEO, F_FULL, F_MASK_BCE, F_FULL_BCE, F_PM, F_PM_EXTENT, F_CENTROID, F_Z, F_Z_ABS = (1 << i for i in range(9))
MASK_GT = ("trunc", "visib", "obj")


def _opt(node, key, default=None):
    if isinstance(node, dict):
        return node.get(key, default)
    return getattr(node, key, default)


def _reject(name, value, allowed):
    raise NotImplementedError(f"{name}={value!r} is not supported (only {', '.join(map(repr, allowed))})")


class Plan:
    """What one config asks of the loss: the active terms as kernel flags, the weights, the GT mask each term uses."""

    def __init__(self, flags, weights, mask_gt, keys):
        self.flags, self.weights, self.mask_gt, self.keys = flags, weights, mask_gt, keys


def check_cfg(cfg):
    """The loss options this implementation covers, as a Plan; anything else is rejected by name."""
    net = cfg.MODEL.POSE_NET
    geo, pnp, loss = net.GEO_HEAD, net.PNP_NET, net.LOSS_CFG
    flags, keys = 0, []
    w = [0.0] * 7
    mask_gt = {}
    if not _opt(geo, "FREEZE", False):
        flags |= F_GEO
        if loss.XYZ_LOSS_TYPE != "L1":
            _reject("XYZ_LOSS_TYPE", loss.XYZ_LOSS_TYPE, ("L1",))
        if loss.XYZ_LOSS_MASK_GT not in MASK_GT:
            _reject("XYZ_LOSS_MASK_GT", loss.XYZ_LOSS_MASK_GT, MASK_GT)
        if loss.MASK_LOSS_TYPE not in ("L1", "BCE"):
            _reject("MASK_LOSS_TYPE", loss.MASK_LOSS_TYPE, ("L1", "BCE"))
        if loss.MASK_LOSS_GT not in MASK_GT + ("full",):
            _reject("MASK_LOSS_GT", loss.MASK_LOSS_GT, MASK_GT + ("full",))
        if loss.REGION_LOSS_TYPE != "CE":
            _reject("REGION_LOSS_TYPE", loss.REGION_LOSS_TYPE, ("CE",))
        if loss.REGION_LOSS_MASK_GT not in MASK_GT:
            _reject("REGION_LOSS_MASK_GT", loss.REGION_LOSS_MASK_GT, MASK_GT)
        flags |= F_MASK_BCE if loss.MASK_LOSS_TYPE == "BCE" else 0
        w[0], w[1], w[3] = float(loss.XYZ_LW), float(loss.MASK_LW), float(loss.REGION_LW)
        mask_gt = {"xyz": loss.XYZ_LOSS_MASK_GT, "mask": loss.MASK_LOSS_GT, "region": loss.REGION_LOSS_MASK_GT}
        keys += ["loss_coor_x", "loss_coor_y", "loss_coor_z", "loss_mask"]
        if loss.FULL_MASK_LW > 0:
            if loss.FULL_MASK_LOSS_TYPE not in ("L1", "BCE"):
                _reject("FULL_MASK_LOSS_TYPE", loss.FULL_MASK_LOSS_TYPE, ("L1", "BCE"))
            flags |= F_FULL | (F_FULL_BCE if loss.FULL_MASK_LOSS_TYPE == "BCE" else 0)
            w[2] = float(loss.FULL_MASK_LW)
            keys.append("loss_mask_full")
        keys.append("loss_region")
    if loss.PM_LW > 0:
        if not loss.PM_R_ONLY:
            _reject("PM_R_ONLY", loss.PM_R_ONLY, (True,))
        if str(loss.PM_LOSS_TYPE).lower() != "l1":
            _reject("PM_LOSS_TYPE", loss.PM_LOSS_TYPE, ("L1",))
        flags |= F_PM | (F_PM_EXTENT if loss.PM_NORM_BY_EXTENT else 0)
        w[4] = float(loss.PM_LW)
        keys.append("loss_PM_R")
    for name in ("ROT_LW", "TRANS_LW", "BIND_LW"):
        if _opt(loss, name, 0.0) > 0:
            _reject(name, _opt(loss, name), (0,))
    if loss.CENTROID_LW > 0:
        if pnp.TRANS_TYPE != "centroid_z":
            _reject("PNP_NET.TRANS_TYPE (with CENTROID_LW > 0)", pnp.TRANS_TYPE, ("centroid_z",))
        if loss.CENTROID_LOSS_TYPE != "L1":
            _reject("CENTROID_LOSS_TYPE", loss.CENTROID_LOSS_TYPE, ("L1",))
        flags |= F_CENTROID
        w[5] = float(loss.CENTROID_LW)
        keys.append("loss_centroid")
    if loss.Z_LW > 0:
        if pnp.Z_TYPE not in ("REL", "ABS"):
            _reject("PNP_NET.Z_TYPE", pnp.Z_TYPE, ("REL", "ABS"))
        if loss.Z_LOSS_TYPE != "L1":
            _reject("Z_LOSS_TYPE", loss.Z_LOSS_TYPE, ("L1",))
        flags |= F_Z | (F_Z_ABS if pnp.Z_TYPE == "ABS" else 0)
        w[6] = float(loss.Z_LW)
        keys.append("loss_z")
    return Plan(flags, w, mask_gt, keys)


def workspace_layout(B, HW):
    """(total bytes, {name: byte offset from the 256-aligned workspace base}) of a call's workspace."""
    L = _lib.lib()
    offs = (_lib.c_size_t * len(LAYOUT_NAMES))()
    _lib.check(L.gdrn_loss_layout(B, HW, offs), "gdrn_loss_layout")
    return L.gdrn_loss_workspace_bytes(B, HW), dict(zip(LAYOUT_NAMES, offs))


def workspace_view(ws, offsets, name, dtype, shape):
    """A stage result the forward left in its workspace, as a tensor view."""
    base = (-ws.data_ptr()) % 256
    n = 1
    for s in shape:
        n *= s
    nbytes = n * torch.empty((), dtype=dtype).element_size()
    o = base + offsets[name]
    return ws[o:o + nbytes].view(dtype).view(*shape)


# ---- symmetry tables: one device table per device, grown as new per-object arrays appear
_SYM_ROWS = {}    # (id(obj), device) -> (obj, first row, K); holding obj keeps its id unique
_SYM_TABLE = {}   # device -> [T, 3, 3] f32


def sym_ranges(sym_infos, B, device):
    """(table [T,3,3] f32, ranges [B,2] i32 = (first row, count)) for the ROIs' symmetry arrays, or (None, None) when no
    ROI has one.  Arrays seen before are not uploaded again."""
    key_dev = str(device)
    table = _SYM_TABLE.get(key_dev)
    T = 0 if table is None else table.shape[0]
    rng = np.zeros((B, 2), np.int32)
    new = []
    for b, s in enumerate(sym_infos):
        if s is None:
            continue
        e = _SYM_ROWS.get((id(s), key_dev))
        if e is None:
            a = s.detach().cpu().numpy() if torch.is_tensor(s) else np.asarray(s)
            a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 3, 3)   # get_closest_rot takes one 3x3 too
            e = (s, T, a.shape[0])
            _SYM_ROWS[(id(s), key_dev)] = e
            new.append(a)
            T += a.shape[0]
        rng[b] = e[1:]
    if new:
        up = torch.from_numpy(np.concatenate(new, 0)).to(device)
        table = up if table is None else torch.cat([table, up], 0)
        _SYM_TABLE[key_dev] = table
    if not rng[:, 1].any():
        return None, None
    return table, torch.from_numpy(rng).to(device)


def _plane(t, name, B, H, W):
    """A [B,1,H,W] head output whose planes are contiguous (a channel slice of the head's output qualifies as is)."""
    if tuple(t.shape) != (B, 1, H, W):
        raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {(B, 1, H, W)}")
    if t.stride(3) != 1 or t.stride(2) != W:
        t = t.contiguous()
    return t


def _f32(t, name):
    if not t.is_cuda:
        raise _lib.GdrnError(f"gdrn_loss needs CUDA tensors (no CPU fallback): {name} is on {t.device}")
    if t.dtype != torch.float32:
        raise TypeError(f"gdrn_loss computes in fp32: {name} is {t.dtype}")
    return t


class Inputs:
    """The kernel's 22 input pointers (csrc/gdrn_loss.cu IN_*), the five batch strides and the sizes of one call."""

    def __init__(self, plan, d):
        self.plan, self.t = plan, d
        self.B, self.HW, self.R1, self.N = d["B"], d["HW"], d["R1"], d["N"]
        order = ("out_x", "out_y", "out_z", "out_mask_vis", "out_mask_full", "m_xyz", "m_mask", "m_full", "m_region",
                 "gt_xyz", "out_region", "gt_region", "out_rot", "gt_rot", "gt_points", "extents", "sym_table",
                 "sym_range", "out_centroid", "out_trans_z", "gt_trans_ratio", "gt_trans")
        self.ptrs = (_lib.c_void_p * len(order))(*[_lib.ptr(d.get(k)) for k in order])
        self.bs = (_lib.c_int64 * 5)(*[d[k].stride(0) if d.get(k) is not None else 0
                                       for k in ("out_x", "out_y", "out_z", "out_mask_vis", "out_mask_full")])
        self.w = (_lib.c_float * 7)(*plan.weights)


def forward_raw(inp):
    """One forward call -> (workspace, offsets)."""
    nb, offs = workspace_layout(inp.B, inp.HW)
    ws = torch.empty(nb, dtype=torch.uint8, device=inp.t["device"])
    _lib.check(_lib.lib().gdrn_loss_forward(inp.ptrs, inp.bs, inp.w, inp.B, inp.HW, inp.R1, inp.N, inp.plan.flags,
                                            _lib.ptr(ws), ws.numel(), _lib.current_stream()), "gdrn_loss_forward")
    return ws, offs


def backward_raw(inp, ws, grad_losses):
    """The gradients of the differentiable inputs (None where a term is off) for upstream gradients [9] f32."""
    d, f = inp.t, inp.plan.flags
    geo = bool(f & F_GEO)
    like = lambda k, on: torch.empty(d[k].shape, dtype=torch.float32, device=d["device"]) if on else None  # noqa: E731
    grads = [like("out_x", geo), like("out_y", geo), like("out_z", geo), like("out_mask_vis", geo),
             like("out_mask_full", f & F_FULL), like("out_region", geo), like("out_rot", f & F_PM),
             like("out_centroid", f & F_CENTROID), like("out_trans_z", f & F_Z)]
    g = grad_losses.to(torch.float32).contiguous()
    gp = (_lib.c_void_p * 9)(*[_lib.ptr(t) for t in grads])
    _lib.check(_lib.lib().gdrn_loss_backward(inp.ptrs, inp.bs, inp.w, inp.B, inp.HW, inp.R1, inp.N, f, _lib.ptr(g), gp,
                                             _lib.ptr(ws), ws.numel(), _lib.current_stream()), "gdrn_loss_backward")
    return grads


class _GdrnLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, inp, out_x, out_y, out_z, out_mask_vis, out_mask_full, out_region, out_rot, out_centroid,
                out_trans_z):
        ws, offs = forward_raw(inp)
        res = workspace_view(ws, offs, "result", torch.float32, (10,))
        # CrossEntropyLoss rejects a target outside [0, R]: one flag read back per call
        if inp.plan.flags & F_GEO and res[9].item() != 0:
            raise ValueError(f"gt_region holds a label outside [0, {inp.R1 - 1}] inside the region mask")
        ctx.inp, ctx.ws = inp, ws
        return res[:9].clone()

    @staticmethod
    def backward(ctx, grad_losses):
        return (None, *backward_raw(ctx.inp, ctx.ws, grad_losses))


def gdrn_loss(model, cfg, out_mask_vis, out_mask_full, gt_mask_trunc, gt_mask_visib, gt_mask_obj, gt_mask_full, out_x,
              out_y, out_z, gt_xyz, gt_xyz_bin, out_region, gt_region, out_rot=None, gt_rot=None, out_trans=None,
              gt_trans=None, out_centroid=None, out_trans_z=None, gt_trans_ratio=None, gt_points=None, sym_infos=None,
              extents=None):
    """GDRN_DoubleMask.gdrn_loss on the GPU -> {loss name: 0-d fp32 tensor}, the reference's keys for ``cfg``.
    ``gt_xyz_bin`` and ``out_trans`` are not used by the supported options."""
    plan = check_cfg(cfg)
    loss_cfg = cfg.MODEL.POSE_NET.LOSS_CFG
    f = plan.flags
    d = {"B": 0, "HW": 1, "R1": 1, "N": 0}
    if f & F_GEO:
        B, _, H, W = out_x.shape
        d.update(B=B, HW=H * W, device=out_x.device)
        for name, t in (("out_x", out_x), ("out_y", out_y), ("out_z", out_z), ("out_mask_vis", out_mask_vis)):
            d[name] = _plane(_f32(t, name), name, B, H, W)
        if f & F_FULL:
            d["out_mask_full"] = _plane(_f32(out_mask_full, "out_mask_full"), "out_mask_full", B, H, W)
        gt_masks = {"trunc": gt_mask_trunc, "visib": gt_mask_visib, "obj": gt_mask_obj, "full": gt_mask_full}
        for role, which in list(plan.mask_gt.items()) + ([("full", "full")] if f & F_FULL else []):
            m = _f32(gt_masks[which], f"gt_mask_{which}")
            if tuple(m.shape) != (B, H, W):
                raise ValueError(f"gt_mask_{which} has shape {tuple(m.shape)}, expected {(B, H, W)}")
            d["m_" + role] = m.contiguous()
        if tuple(gt_xyz.shape) != (B, 3, H, W):
            raise ValueError(f"gt_xyz has shape {tuple(gt_xyz.shape)}, expected {(B, 3, H, W)}")
        d["gt_xyz"] = _f32(gt_xyz, "gt_xyz").contiguous()
        if out_region.dim() != 4 or out_region.shape[0] != B or tuple(out_region.shape[2:]) != (H, W):
            raise ValueError(f"out_region has shape {tuple(out_region.shape)}, expected {(B, 'R+1', H, W)}")
        d["out_region"] = _f32(out_region, "out_region").contiguous()
        d["R1"] = out_region.shape[1]
        if tuple(gt_region.shape) != (B, H, W):
            raise ValueError(f"gt_region has shape {tuple(gt_region.shape)}, expected {(B, H, W)}")
        d["gt_region"] = gt_region.to(device=out_x.device).long().contiguous()
    if f & F_PM:
        if gt_rot is None or gt_points is None or out_rot is None:
            raise ValueError("point matching needs out_rot, gt_rot and gt_points")
        if gt_rot.shape[-1] == 4:
            raise NotImplementedError("gt_rot as quaternions [B,4] is not supported (only rotation matrices [B,3,3])")
        B = out_rot.shape[0]
        d.update(B=B, device=out_rot.device)
        d["out_rot"] = _f32(out_rot, "out_rot").contiguous()
        d["gt_rot"] = _f32(gt_rot, "gt_rot").contiguous()
        d["gt_points"] = _f32(gt_points, "gt_points").contiguous()
        if tuple(d["out_rot"].shape) != (B, 3, 3) or tuple(d["gt_rot"].shape) != (B, 3, 3):
            raise ValueError("out_rot and gt_rot must be [B,3,3]")
        if d["gt_points"].dim() != 3 or d["gt_points"].shape[0] != B or d["gt_points"].shape[2] != 3:
            raise ValueError(f"gt_points has shape {tuple(gt_points.shape)}, expected [B,N,3]")
        d["N"] = d["gt_points"].shape[1]
        if f & F_PM_EXTENT:
            d["extents"] = _f32(extents, "extents").contiguous()
        if loss_cfg.PM_LOSS_SYM:
            if sym_infos is None or len(sym_infos) != B:
                raise ValueError("PM_LOSS_SYM needs one sym_infos entry (array or None) per ROI")
            d["sym_table"], d["sym_range"] = sym_ranges(sym_infos, B, d["device"])
    if f & F_CENTROID:
        d.setdefault("device", out_centroid.device)
        d["B"] = out_centroid.shape[0]
        d["out_centroid"] = _f32(out_centroid, "out_centroid").contiguous()
        d["gt_trans_ratio"] = _f32(gt_trans_ratio, "gt_trans_ratio").contiguous()
    if f & F_Z:
        d.setdefault("device", out_trans_z.device)
        d["B"] = out_trans_z.shape[0]
        d["out_trans_z"] = _f32(out_trans_z, "out_trans_z").contiguous()
        if f & F_Z_ABS:
            d["gt_trans"] = _f32(gt_trans, "gt_trans").contiguous()
        else:
            d["gt_trans_ratio"] = _f32(gt_trans_ratio, "gt_trans_ratio").contiguous()
    if "device" not in d:
        return {}
    inp = Inputs(plan, d)
    with torch.cuda.device(d["device"]):
        res = _GdrnLoss.apply(inp, *[d.get(k) for k in ("out_x", "out_y", "out_z", "out_mask_vis", "out_mask_full",
                                                           "out_region", "out_rot", "out_centroid", "out_trans_z")])
    vals = dict(zip(RESULT_KEYS, res.unbind(0)))
    loss_dict = {k: vals[k] for k in plan.keys}
    if cfg.MODEL.POSE_NET.USE_MTL:
        for k in loss_dict:
            lv = getattr(model, k.replace("loss_", "log_var_"))
            loss_dict[k] = loss_dict[k] * torch.exp(-lv) + torch.log(1 + torch.exp(lv))
    return loss_dict
