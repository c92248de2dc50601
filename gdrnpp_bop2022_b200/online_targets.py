"""Online training-target rendering on the GPU (SURVEY.md §8f rank 3).

Mirrors the XYZ_BP branch of ``batch_data`` (core/gdrn_modeling/engine/engine_utils.py:131-187): render every ROI's depth
(the reference loops over ROIs calling the EGL renderer; here ONE launch of the CUDA rasteriser over the mesh registry),
back-project to object space (``misc.calc_xyz_bp_batch``, lib/pysixd/misc.py:412-457), derive ``roi_mask_obj``, the region
labels (``xyz_to_region_batch``, core/utils/data_utils.py:283-301) and the normalised ``roi_xyz``.  No EGL / GL, no CPU
fallback.
"""
import torch

from . import _lib
from .renderer import render_meshes


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


@_lib.on_device(0)
def xyz_region_targets(depth, R, T, K, fps_points=None, extents=None, want_xyz_raw=False):
    """depth [n,H,W], R [n,3,3], T [n,3], K [n,3,3] (CUDA) -> dict with ``roi_mask_obj`` [n,H,W] and, when given the inputs
    they need, ``roi_xyz`` [n,3,H,W] (extents), ``roi_region`` [n,H,W] int64 (fps_points [n,F,3]), ``xyz`` [n,H,W,3]."""
    if not depth.is_cuda:
        raise _lib.GdrnError("xyz_region_targets needs CUDA tensors (no CPU fallback)")
    dev = depth.device
    n, H, W = depth.shape
    d, Rm, Tm, Km = _f32(depth, dev), _f32(R, dev).reshape(n, 9), _f32(T, dev).reshape(n, 3), _f32(K, dev).reshape(n, 9)
    out = {"roi_mask_obj": torch.empty((n, H, W), dtype=torch.float32, device=dev)}
    fps = ext = None
    F = 0
    if fps_points is not None:
        fps = _f32(fps_points, dev)
        F = fps.shape[1]
        out["roi_region"] = torch.empty((n, H, W), dtype=torch.int64, device=dev)
    if extents is not None:
        ext = _f32(extents, dev).reshape(n, 3)
        out["roi_xyz"] = torch.empty((n, 3, H, W), dtype=torch.float32, device=dev)
    if want_xyz_raw:
        out["xyz"] = torch.empty((n, H, W, 3), dtype=torch.float32, device=dev)
    if n:
        _lib.check(_lib.lib().gdrn_xyz_region_targets(_lib.ptr(d), _lib.ptr(Rm), _lib.ptr(Tm), _lib.ptr(Km), _lib.ptr(fps), _lib.ptr(ext),
                                                      n, H, W, F, _lib.ptr(out.get("roi_xyz")), _lib.ptr(out.get("xyz")),
                                                      _lib.ptr(out["roi_mask_obj"]), _lib.ptr(out.get("roi_region")),
                                                      _lib.current_stream()), "gdrn_xyz_region_targets")
    return out


def calc_xyz_bp_batch(depth, R, T, K, fmt="BHWC"):
    """lib/pysixd/misc.py:412-457: depth [B,H,W], R [B,3,3], T [B,3], K [B,3,3] -> xyz [B,H,W,3] (or [B,3,H,W])."""
    xyz = xyz_region_targets(depth, R, T, K, want_xyz_raw=True)["xyz"]
    return xyz if fmt == "BHWC" else xyz.permute(0, 3, 1, 2).contiguous()


def xyz_to_region_batch(xyz, fps_points, mask=None):
    """core/utils/data_utils.py:283-301 for an arbitrary xyz map [b,h,w,3] (CUDA): nearest fps point (1..F), 0 = background.
    The generic entry (torch.cdist on the device, like the reference); the training path uses the fused kernel
    (xyz_region_targets / render_roi_targets), which labels the pixels while it back-projects them."""
    b, h, w, _ = xyz.shape
    d = torch.cdist(xyz.reshape(b, -1, 3).float(), fps_points.float(), p=2)
    region = d.argmin(-1).view(b, h, w) + 1
    if mask is None:
        mask = ((xyz[..., 0] != 0) & (xyz[..., 1] != 0) & (xyz[..., 2] != 0)).to(torch.float32)
    return (region * mask).to(torch.long)


def render_roi_targets(models, roi_cls, ego_rot, trans, roi_zoom_K, roi_extent, roi_fps_points=None, out_res=64, znear=0.1,
                       zfar=100.0):
    """The rendering block of batch_data (engine_utils.py:131-187) for a whole batch: models = list of Model3D indexed by
    roi_cls.  Returns roi_xyz, roi_mask_obj, roi_region (when fps points are given) and the rendered roi_depth; two
    launches (rasteriser + target kernel), no host loop over ROIs, no sync."""
    dev = ego_rot.device
    with torch.cuda.device(dev):
        reg = torch.tensor([m.mesh_id for m in models], dtype=torch.int32, device=dev)
        ids = reg[roi_cls.to(device=dev, dtype=torch.long)].contiguous()
        poses = torch.cat([ego_rot.float(), trans.float().reshape(-1, 3, 1)], dim=2).contiguous()
        depth = render_meshes(ids, poses, roi_zoom_K, out_res, out_res, znear, zfar)
        out = xyz_region_targets(depth, ego_rot, trans, roi_zoom_K, fps_points=roi_fps_points, extents=roi_extent)
    out["roi_depth"] = depth
    return out
