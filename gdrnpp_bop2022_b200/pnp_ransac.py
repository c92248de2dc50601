"""Batched GPU RANSAC-PnP behind the reference's TEST.USE_PNP surfaces.

Mirrors ``get_pnp_ransac_pose`` / ``get_img_model_points_with_coords2d`` (core/gdrn_modeling/engine/gdrn_evaluator.py:
1122-1221) and ``misc.pnp_v2(..., ransac=True, ransac_reprojErr=3, ransac_iter=100)`` (lib/pysixd/misc.py:153-208), for all
ROIs of a batch in one launch of libgdrn_b200.so (csrc/pnp_ransac.cu), and the network-initialised TEST.PNP_TYPE
variants of ``process_net_and_pnp`` (gdrn_evaluator.py:241-371).  No CPU fallback.
"""
import torch

from . import _lib


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


@_lib.on_device(0)
def pnp_ransac_from_maps(coor_x, coor_y, coor_z, mask, roi_coord_2d, im_H, im_W, roi_extents, cams, mask_thr=0.5,
                         reproj_err=3.0, iters=100, seed=0, idxs=None, return_inliers=False):
    """coor_x/y/z, mask: [n,1,hw,hw] raw outputs of GDRN_DoubleMask.forward; roi_coord_2d [n,2,hw,hw]; im_H, im_W [n];
    roi_extents [n,3]; cams [n,3,3] -> poses [n,3,4] (R|t; -100 where the reference returns its sentinel)."""
    if not coor_x.is_cuda:
        raise _lib.GdrnError("pnp_ransac_from_maps needs CUDA tensors (no CPU fallback)")
    dev = coor_x.device
    n, hw = coor_x.shape[0], coor_x.shape[-1]
    cx, cy, cz, m, c2d = (_f32(t, dev) for t in (coor_x, coor_y, coor_z, mask, roi_coord_2d))
    im_hw = torch.stack([torch.as_tensor(im_H, dtype=torch.float32).reshape(-1), torch.as_tensor(im_W, dtype=torch.float32).reshape(-1)], dim=1)
    im_hw = _f32(im_hw, dev)
    ext, Ks = _f32(roi_extents, dev), _f32(cams, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    poses = torch.empty((n, 3, 4), dtype=torch.float32, device=dev)
    ninl = torch.empty((n,), dtype=torch.int32, device=dev)
    imask = torch.empty((n, hw * hw), dtype=torch.uint8, device=dev) if return_inliers else None
    ix = None if idxs is None else idxs.detach().to(device=dev, dtype=torch.int32).contiguous()
    if ix is not None:
        iters = ix.shape[1]
    if n > 0:
        _lib.check(_lib.lib().gdrn_pnp_ransac_maps(_lib.ptr(cx), _lib.ptr(cy), _lib.ptr(cz), _lib.ptr(m), _lib.ptr(c2d), _lib.ptr(im_hw),
                                                   _lib.ptr(ext), _lib.ptr(Ks), _lib.ptr(ix), n, hw, int(iters), float(mask_thr),
                                                   float(reproj_err), int(seed) & 0xFFFFFFFF, _lib.ptr(poses), _lib.ptr(ninl),
                                                   _lib.ptr(imask), _lib.current_stream()), "gdrn_pnp_ransac_maps")
    return (poses, ninl, imask.view(n, hw, hw)) if return_inliers else poses


@_lib.on_device(0)
def solve_pnp_ransac(pts3d, pts2d, cams, reproj_err=3.0, iters=100, seed=0, idxs=None, return_inliers=False):
    """Explicit correspondences: pts3d [n,npts,3], pts2d [n,npts,2], cams [n,3,3] (CUDA) -> poses [n,3,4]
    (the batched stand-in for n calls of misc.pnp_v2(points_3d, points_2d, K, ransac=True))."""
    if not pts3d.is_cuda:
        raise _lib.GdrnError("solve_pnp_ransac needs CUDA tensors (no CPU fallback)")
    dev = pts3d.device
    n, npts = pts3d.shape[0], pts3d.shape[1]
    p3, p2, Ks = _f32(pts3d, dev), _f32(pts2d, dev), _f32(cams, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    poses = torch.empty((n, 3, 4), dtype=torch.float32, device=dev)
    ninl = torch.empty((n,), dtype=torch.int32, device=dev)
    imask = torch.empty((n, npts), dtype=torch.uint8, device=dev) if return_inliers else None
    ix = None if idxs is None else idxs.detach().to(device=dev, dtype=torch.int32).contiguous()
    if ix is not None:
        iters = ix.shape[1]
    _lib.check(_lib.lib().gdrn_pnp_ransac_points(_lib.ptr(p3), _lib.ptr(p2), _lib.ptr(Ks), _lib.ptr(ix), n, npts, int(iters),
                                                 float(reproj_err), int(seed) & 0xFFFFFFFF, _lib.ptr(poses), _lib.ptr(ninl),
                                                 _lib.ptr(imask), _lib.current_stream()), "gdrn_pnp_ransac_points")
    return (poses, ninl, imask) if return_inliers else poses


@_lib.on_device(0)
def pnp_ransac_trace(pts3d=None, pts2d=None, cams=None, maps=None, mask_thr=0.5, reproj_err=3.0, iters=100, seed=0,
                     idxs=None):
    """The RANSAC-PnP kernel with a record of every stage (gdrn_pnp_ransac_trace), for tests.  Give either the points
    form (pts3d [n,npts,3], pts2d [n,npts,2]) or the maps form, ``maps`` = the first eight arguments of
    pnp_ransac_from_maps (coor_x, coor_y, coor_z, mask, roi_coord_2d, im_H, im_W, roi_extents); cams [n,3,3].
    Returns a dict of tensors on the device: poses [n,3,4], n_inliers [n], inlier_mask [n,npts] (as the production
    entries return them) and N [n], src [n,4096], samples [n,iters,4], nsol [n,iters], hyp [n,iters,3,4] f64,
    cnt [n,iters], best [n], inl [n,2,4096] bool, round_pose [n,2,2,3,4] f64 (start, end), round_cost [n,2,3] f64
    (start, lowest evaluated, returned), pose [n,3,4] f64.  Entries a ROI does not reach hold -1 / NaN / False."""
    ref = pts3d if maps is None else maps[0]
    if not ref.is_cuda:
        raise _lib.GdrnError("pnp_ransac_trace needs CUDA tensors (no CPU fallback)")
    dev = ref.device
    n = ref.shape[0]
    if maps is None:
        npts = pts3d.shape[1]
        p3, p2 = _f32(pts3d, dev), _f32(pts2d, dev)
        cx = cy = cz = m = c2d = im_hw = ext = None
    else:
        coor_x, coor_y, coor_z, mask, roi_coord_2d, im_H, im_W, roi_extents = maps
        npts = coor_x.shape[-1] * coor_x.shape[-2]
        p3 = p2 = None
        cx, cy, cz, m, c2d = (_f32(t, dev) for t in (coor_x, coor_y, coor_z, mask, roi_coord_2d))
        im_hw = _f32(torch.stack([torch.as_tensor(im_H, dtype=torch.float32).reshape(-1),
                                  torch.as_tensor(im_W, dtype=torch.float32).reshape(-1)], dim=1), dev)
        ext = _f32(roi_extents, dev)
    Ks = _f32(cams, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    ix = None if idxs is None else idxs.detach().to(device=dev, dtype=torch.int32).contiguous()
    if ix is not None:
        iters = ix.shape[1]
    i32 = lambda *s: torch.full(s, -1, dtype=torch.int32, device=dev)
    f64 = lambda *s: torch.full(s, float("nan"), dtype=torch.float64, device=dev)
    out = dict(poses=torch.empty((n, 3, 4), dtype=torch.float32, device=dev), n_inliers=torch.empty((n,), dtype=torch.int32, device=dev),
               inlier_mask=torch.empty((n, npts), dtype=torch.uint8, device=dev), N=i32(n), src=i32(n, 4096),
               samples=i32(n, iters, 4), nsol=i32(n, iters), hyp=f64(n, iters, 3, 4), cnt=i32(n, iters), best=i32(n),
               inl=torch.zeros((n, 2, 4096), dtype=torch.uint8, device=dev), round_pose=f64(n, 2, 2, 3, 4),
               round_cost=f64(n, 2, 3), pose=f64(n, 3, 4))
    P = lambda k: _lib.ptr(out[k])
    _lib.check(_lib.lib().gdrn_pnp_ransac_trace(_lib.ptr(cx), _lib.ptr(cy), _lib.ptr(cz), _lib.ptr(m), _lib.ptr(c2d), _lib.ptr(im_hw),
                                                _lib.ptr(ext), _lib.ptr(p3), _lib.ptr(p2), _lib.ptr(Ks), _lib.ptr(ix), n, npts,
                                                int(iters), float(mask_thr), float(reproj_err), int(seed) & 0xFFFFFFFF,
                                                P("poses"), P("n_inliers"), P("inlier_mask"), P("N"), P("src"), P("samples"),
                                                P("nsol"), P("hyp"), P("cnt"), P("best"), P("inl"), P("round_pose"),
                                                P("round_cost"), P("pose"), _lib.current_stream()), "gdrn_pnp_ransac_trace")
    out["inl"] = out["inl"].bool()
    return out


# TEST.PNP_TYPE -> pnp_type of gdrn_pnp_net_maps (gdrn_evaluator.py:164-175); "ransac_pnp" is pnp_ransac_from_maps
PNP_NET_TYPES = {"net_iter_pnp": 0, "net_ransac_pnp": 1, "net_ransac_pnp_rot": 2}


@_lib.on_device(0)
def pnp_net_from_maps(coor_x, coor_y, coor_z, mask, roi_coord_2d, im_H, im_W, roi_extents, cams, rot, trans,
                      pnp_type="net_iter_pnp", mask_thr=0.5, reproj_err=3.0, ransac_iters=20, seed=0, return_used=False):
    """The network-initialised post-processes of process_net_and_pnp (gdrn_evaluator.py:241-371) for a whole batch in
    one call, no host sync.  Inputs as pnp_ransac_from_maps plus the network pose rot [n,3,3], trans [n,3].
      net_iter_pnp       LM over all selected correspondences from the network pose (cv2.solvePnP ITERATIVE with
                         useExtrinsicGuess); no translation guard (it never fires in the reference for this type)
      net_ransac_pnp     RANSAC at 20 iterations; t = t_net where ||t - t_net|| > 1 m
      net_ransac_pnp_rot RANSAC rotation, t = t_net
    ROIs with < 4 correspondences, or without a RANSAC model, keep the network pose.  -> poses [n,3,4]
    (and n_used [n] int32 with return_used: the correspondences the pose was fitted to, 0 where the network pose came back)."""
    if pnp_type not in PNP_NET_TYPES:
        raise NotImplementedError(f"pnp_type {pnp_type!r} (network-initialised types: {sorted(PNP_NET_TYPES)})")
    if not coor_x.is_cuda:
        raise _lib.GdrnError("pnp_net_from_maps needs CUDA tensors (no CPU fallback)")
    dev = coor_x.device
    n, hw = coor_x.shape[0], coor_x.shape[-1]
    cx, cy, cz, m, c2d = (_f32(t, dev) for t in (coor_x, coor_y, coor_z, mask, roi_coord_2d))
    im_hw = torch.stack([torch.as_tensor(im_H, dtype=torch.float32).reshape(-1), torch.as_tensor(im_W, dtype=torch.float32).reshape(-1)], dim=1)
    im_hw = _f32(im_hw, dev)
    ext, Ks = _f32(roi_extents, dev), _f32(cams, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    R0, t0 = _f32(rot, dev).reshape(n, 3, 3), _f32(trans, dev).reshape(n, 3)
    poses = torch.empty((n, 3, 4), dtype=torch.float32, device=dev)
    used = torch.empty((n,), dtype=torch.int32, device=dev)
    if n > 0:
        _lib.check(_lib.lib().gdrn_pnp_net_maps(_lib.ptr(cx), _lib.ptr(cy), _lib.ptr(cz), _lib.ptr(m), _lib.ptr(c2d), _lib.ptr(im_hw),
                                                _lib.ptr(ext), _lib.ptr(Ks), _lib.ptr(R0), _lib.ptr(t0), n, hw, PNP_NET_TYPES[pnp_type],
                                                float(mask_thr), float(reproj_err), int(ransac_iters), int(seed) & 0xFFFFFFFF,
                                                _lib.ptr(poses), _lib.ptr(used), _lib.current_stream()), "gdrn_pnp_net_maps")
    return (poses, used) if return_used else poses


@_lib.on_device(0)
def solve_pnp_iterative(pts3d, pts2d, cams, rot0, trans0):
    """Explicit correspondences: pts3d [n,npts,3], pts2d [n,npts,2], cams [n,3,3], initial pose rot0 [n,3,3],
    trans0 [n,3] (CUDA) -> poses [n,3,4]: the batched stand-in for n calls of
    cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) (LM on all points; < 4 points -> the initial pose)."""
    if not pts3d.is_cuda:
        raise _lib.GdrnError("solve_pnp_iterative needs CUDA tensors (no CPU fallback)")
    dev = pts3d.device
    n, npts = pts3d.shape[0], pts3d.shape[1]
    p3, p2, Ks = _f32(pts3d, dev), _f32(pts2d, dev), _f32(cams, dev).reshape(-1, 3, 3)
    if Ks.shape[0] == 1 and n > 1:
        Ks = Ks.expand(n, 3, 3).contiguous()
    R0, t0 = _f32(rot0, dev).reshape(n, 3, 3), _f32(trans0, dev).reshape(n, 3)
    poses = torch.empty((n, 3, 4), dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().gdrn_pnp_iterative_points(_lib.ptr(p3), _lib.ptr(p2), _lib.ptr(Ks), _lib.ptr(R0), _lib.ptr(t0), n, npts,
                                                    _lib.ptr(poses), _lib.current_stream()), "gdrn_pnp_iterative_points")
    return poses
