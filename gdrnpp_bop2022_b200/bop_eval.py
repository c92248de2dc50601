"""BOP19 pose errors as batched GPU calls: VSD, MSSD, MSPD, ADD / ADI (and AD = ADI for symmetric objects, ADD otherwise).

Mirrors the error functions of lib/pysixd/pose_error.py as lib/pysixd/scripts/eval_calc_errors.py calls them, for many
(estimate, GT) pairs per call instead of one pair per numpy call:
  * vsd        pose_error.vsd (:22-128), bop19 visibility, step cost.  Equal to the reference bit for bit given the same
               f32 depth images (rendered estimate / GT depth, test depth in mm), K, taus and delta.
  * mssd_mspd  pose_error.mssd / mspd (:131-179) over the symmetry set of misc.get_symmetry_transformations, one pass.
  * ad         pose_error.add / adi (:256-296); ADI is a brute-force nearest-neighbour search in f64.
  * rt_errors  pose_error.re / te or re_sym / te_sym (:359-437); proj_errors: arp_2d / arp_2d_sym (:183-193, 440-445).
               These serve eval_pose_results_more.py, the counterpart of the reference script of that name.
The gates of eval_calc_errors.py:360-374 are host restatements (sphere_projections_overlap, spheres_overlap) whose
results the calls take per pair.  Units are the BOP ones: points and translations in mm, depth in mm.
No CPU fallback: every call needs CUDA tensors and raises GdrnError otherwise.
"""
import argparse
import json
import math
import os
import sys
import time

if __package__ in (None, ""):   # run by path (python gdrnpp_bop2022_b200/bop_eval.py), as VAL.SCRIPT_PATH is invoked
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    __package__ = "gdrnpp_bop2022_b200"

import numpy as np
import torch

from . import _lib
from ._lib import GdrnError

# dataset_params.get_model_params (lib/pysixd/dataset_params.py:98-132).  For any other dataset an object counts as
# symmetric when its models_info entry lists at least one symmetry.
SYMMETRIC_OBJ_IDS = {
    "lm": [3, 7, 10, 11],
    "lmo": [10, 11],
    "tless": list(range(1, 31)),
    "tudl": [],
    "tyol": [3, 4, 5, 6, 7, 8, 10, 11, 12, 13, 15, 16, 17, 18, 19, 21],
    "ruapc": [8, 9, 12, 13],
    "icmi": [1, 2, 6],
    "icbin": [1],
    "itodd": [2, 3, 4, 5, 7, 8, 9, 11, 12, 14, 17, 18, 19, 23, 24, 25, 27, 28],
    "hbs": [10, 12, 18, 29],
    "hb": [6, 10, 11, 12, 13, 14, 18, 24, 29],
    "ycbv": [1, 13, 14, 16, 18, 19, 20, 21],
    "ycbvposecnn": [13, 16, 19, 20, 21],
}


def is_symmetric(dataset, obj_id, model_info):
    """Whether the `ad` error uses ADI (True) or ADD (False) for this object (eval_calc_errors.py:433-453)."""
    if dataset in SYMMETRIC_OBJ_IDS:
        return int(obj_id) in SYMMETRIC_OBJ_IDS[dataset]
    return bool(model_info.get("symmetries_discrete")) or bool(model_info.get("symmetries_continuous"))


def _rotation_matrix(angle, direction):
    """transform.rotation_matrix (lib/pysixd/transform.py:300-339) about an axis through the origin, 3x3."""
    sina, cosa = math.sin(angle), math.cos(angle)
    d = np.array(direction[:3], dtype=np.float64, copy=True)
    d /= math.sqrt(np.dot(d, d))
    R = np.diag([cosa, cosa, cosa])
    R += np.outer(d, d) * (1.0 - cosa)
    d *= sina
    R += np.array([[0.0, -d[2], d[1]], [d[2], 0.0, -d[0]], [-d[1], d[0], 0.0]])
    return R


def get_symmetry_transformations(model_info, max_sym_disc_step):
    """misc.get_symmetry_transformations (lib/pysixd/misc.py:234-282): the identity, the discrete symmetries and the
    discretised continuous ones (ceil(pi / max_sym_disc_step) steps per axis), combined.  -> list of {'R', 't'} (t 3x1)."""
    trans_disc = [{"R": np.eye(3), "t": np.array([[0, 0, 0]]).T}]
    for sym in model_info.get("symmetries_discrete", []):
        sym_4x4 = np.reshape(sym, (4, 4))
        trans_disc.append({"R": sym_4x4[:3, :3], "t": sym_4x4[:3, 3].reshape((3, 1))})
    trans_cont = []
    for sym in model_info.get("symmetries_continuous", []):
        axis = np.array(sym["axis"])
        offset = np.array(sym["offset"]).reshape((3, 1))
        steps = int(np.ceil(np.pi / max_sym_disc_step))
        step = 2.0 * np.pi / steps
        for i in range(1, steps):
            R = _rotation_matrix(i * step, axis)
            trans_cont.append({"R": R, "t": -(R.dot(offset)) + offset})
    trans = []
    for td in trans_disc:
        if trans_cont:
            for tc in trans_cont:
                trans.append({"R": tc["R"].dot(td["R"]), "t": tc["R"].dot(td["t"]) + tc["t"]})
        else:
            trans.append(td)
    return trans


def sphere_projections_overlap(radius, p1, p2):
    """misc.overlapping_sphere_projections (lib/pysixd/misc.py:1219-1241), the VSD gate."""
    p1, p2 = np.asarray(p1, np.float64).ravel(), np.asarray(p2, np.float64).ravel()
    if p1[2] == 0 or p2[2] == 0:
        return False
    proj_dist = np.linalg.norm((p1 / p1[2])[:2] - (p2 / p2[2])[:2])
    return bool(proj_dist < radius * (1.0 / p1[2] + 1.0 / p2[2]))


def spheres_overlap(t_e, t_g, diameter):
    """eval_calc_errors.py:371-374, the MSSD / AD gate: the centres are closer than the diameter."""
    return bool(np.linalg.norm(np.asarray(t_e, np.float64).reshape(3, 1) - np.asarray(t_g, np.float64).reshape(3, 1))
                < diameter)


def _need_cuda(*ts):
    for t in ts:
        if not (torch.is_tensor(t) and t.is_cuda):
            raise GdrnError("bop_eval needs CUDA tensors (no CPU fallback)")


def _vec(x, n, dtype, dev, what, broadcast=False):
    t = torch.as_tensor(x).to(device=dev, dtype=dtype).reshape(-1).contiguous()
    if broadcast and t.numel() == 1 and n > 1:
        t = t.expand(n).contiguous()
    if t.numel() != n:
        raise GdrnError(f"{what}: expected {n} values, got {t.numel()}")
    return t


def _gate(gate, n, dev, what):
    if gate is None:
        return torch.ones(n, dtype=torch.uint8, device=dev)
    return _vec(gate, n, torch.uint8, dev, what)


def _mats(x, n, shape, dev, what):
    t = torch.as_tensor(x).to(device=dev, dtype=torch.float64).contiguous()
    if t.ndim == len(shape):
        t = t.unsqueeze(0).expand(n, *shape).contiguous()
    if tuple(t.shape) != (n,) + tuple(shape):
        raise GdrnError(f"{what}: expected shape {(n,) + tuple(shape)}, got {tuple(t.shape)}")
    return t


@_lib.on_device(0)
def vsd(depth_est, depth_gt, depth_test, pair_est, pair_gt, pair_img, K, diameter, taus, delta,
        normalized_by_diameter=True, gate=None):
    """VSD of P pairs.  depth_est [Ne,H,W], depth_gt [Ng,H,W], depth_test [Ni,H,W] (f32 CUDA, mm, 0 = none / missing);
    pair p compares depth_est[pair_est[p]] with depth_gt[pair_gt[p]] in image depth_test[pair_img[p]].  K [P,3,3] or
    [3,3], diameter [P] or scalar (mm), taus [T] (T <= 32), delta (mm).  gate [P] (False = sphere projections do not
    overlap -> 1.0 for every tau).  Returns errors [P,T] f64, equal bit for bit to pose_error.vsd on these depths."""
    _need_cuda(depth_est, depth_gt, depth_test)
    dev = depth_est.device
    if depth_est.ndim != 3 or depth_gt.ndim != 3 or depth_test.ndim != 3:
        raise GdrnError("vsd: depth images must be [N,H,W]")
    H, W = depth_est.shape[1:]
    if tuple(depth_gt.shape[1:]) != (H, W) or tuple(depth_test.shape[1:]) != (H, W):
        raise GdrnError("vsd: estimate, GT and test depth images differ in size")
    if any(t.dtype != torch.float32 for t in (depth_est, depth_gt, depth_test)):
        raise GdrnError("vsd: depth images must be float32")
    pe = torch.as_tensor(pair_est).to(device=dev, dtype=torch.int32).reshape(-1).contiguous()
    P = pe.numel()
    if P == 0:
        return torch.empty((0, len(taus)), dtype=torch.float64, device=dev)
    pg = _vec(pair_gt, P, torch.int32, dev, "vsd pair_gt")
    pi = _vec(pair_img, P, torch.int32, dev, "vsd pair_img")
    for idx, n, what in ((pe, depth_est.shape[0], "pair_est"), (pg, depth_gt.shape[0], "pair_gt"),
                         (pi, depth_test.shape[0], "pair_img")):
        if bool(((idx < 0) | (idx >= n)).any()):
            raise GdrnError(f"vsd: {what} out of range [0, {n})")
    Ks = _mats(K, P, (3, 3), dev, "vsd K")
    diam = _vec(diameter, P, torch.float64, dev, "vsd diameter", broadcast=True)
    g = _gate(gate, P, dev, "vsd gate")
    taus_t = torch.as_tensor(np.asarray(taus, np.float64)).to(dev).contiguous()
    T = taus_t.numel()
    L = _lib.lib()
    ws_bytes = L.gdrn_vsd_workspace_bytes(P, T)
    ws = torch.empty((max(ws_bytes, 8) + 7) // 8, dtype=torch.int64, device=dev)
    errors = torch.empty((P, T), dtype=torch.float64, device=dev)
    de, dg, dt = depth_est.contiguous(), depth_gt.contiguous(), depth_test.contiguous()
    _lib.check(L.gdrn_vsd_errors(_lib.ptr(de), _lib.ptr(dg), _lib.ptr(dt), H, W, _lib.ptr(pe), _lib.ptr(pg), _lib.ptr(pi),
                                 _lib.ptr(Ks), _lib.ptr(diam), _lib.ptr(g), P, _lib.ptr(taus_t), T, float(delta),
                                 int(bool(normalized_by_diameter)), _lib.ptr(ws), ws.numel() * 8, _lib.ptr(errors),
                                 _lib.current_stream()), "gdrn_vsd_errors")
    return errors


class PoseErrorModels:
    """The model points (models_eval, mm) and symmetry sets of a dataset's objects, packed on the GPU once.

    points: {obj_id: [N,3]}; model_infos: {obj_id: models_info entry} (diameter, symmetries)."""

    def __init__(self, points, model_infos, max_sym_disc_step=0.01, device="cuda"):
        self.device = torch.device(device)
        self.obj_ids = sorted(int(o) for o in points)
        self.slot = {o: i for i, o in enumerate(self.obj_ids)}
        pts = [np.asarray(points[o], np.float64).reshape(-1, 3) for o in self.obj_ids]
        if any(len(p) == 0 for p in pts):
            raise GdrnError("PoseErrorModels: an object has no points")
        syms = []
        for o in self.obj_ids:
            info = model_infos[o]
            syms.append(np.stack([np.hstack([np.asarray(s["R"], np.float64), np.asarray(s["t"], np.float64).reshape(3, 1)])
                                  for s in get_symmetry_transformations(info, max_sym_disc_step)]))
        self.diameters = {o: float(model_infos[o]["diameter"]) for o in self.obj_ids}
        self.n_pts = [len(p) for p in pts]
        self.n_syms = [len(s) for s in syms]
        self.pts = torch.from_numpy(np.concatenate(pts)).to(self.device).contiguous()
        self.syms = torch.from_numpy(np.concatenate(syms)).to(self.device).contiguous()
        self.pt_offsets = torch.tensor(np.concatenate([[0], np.cumsum(self.n_pts)]), dtype=torch.int64, device=self.device)
        self.sym_offsets = torch.tensor(np.concatenate([[0], np.cumsum(self.n_syms)]), dtype=torch.int64,
                                        device=self.device)

    def slots(self, obj_ids):
        try:
            return [self.slot[int(o)] for o in np.asarray(obj_ids).reshape(-1)]
        except KeyError as e:
            raise GdrnError(f"PoseErrorModels: unknown obj_id {e.args[0]}") from None


def _poses(R, t, P, dev, what):
    R = _mats(R, P, (3, 3), dev, what + " R")
    t = torch.as_tensor(t).to(device=dev, dtype=torch.float64)
    if t.numel() != 3 * P:
        raise GdrnError(f"{what} t: expected {P} translations, got {t.numel()} values")
    return torch.cat([R, t.reshape(P, 3, 1)], dim=2).contiguous()


def mssd_mspd(models, obj_ids, R_est, t_est, R_gt, t_gt, K, gate_mssd=None):
    """MSSD (mm) and MSPD (px) of P pairs; pair p is object obj_ids[p] of `models` (PoseErrorModels).  R [P,3,3],
    t [P,3] (mm), K [P,3,3] or [3,3].  gate_mssd [P] (False = spheres do not overlap -> MSSD inf; MSPD has no gate).
    Returns (mssd [P], mspd [P]) f64 CUDA tensors."""
    dev = models.device
    slots = models.slots(obj_ids)
    P = len(slots)
    if P == 0:
        e = torch.empty(0, dtype=torch.float64, device=dev)
        return e, e.clone()
    with torch.cuda.device(dev):
        po = torch.tensor(slots, dtype=torch.int32, device=dev)
        pose_e, pose_g = _poses(R_est, t_est, P, dev, "mssd_mspd est"), _poses(R_gt, t_gt, P, dev, "mssd_mspd gt")
        Ks = _mats(K, P, (3, 3), dev, "mssd_mspd K")
        g = _gate(gate_mssd, P, dev, "mssd_mspd gate")
        max_syms = max(models.n_syms[s] for s in set(slots))
        mssd = torch.empty(P, dtype=torch.float64, device=dev)
        mspd = torch.empty(P, dtype=torch.float64, device=dev)
        _lib.check(_lib.lib().gdrn_sym_max_dist(_lib.ptr(models.pts), _lib.ptr(models.pt_offsets), _lib.ptr(models.syms),
                                                _lib.ptr(models.sym_offsets), _lib.ptr(po), _lib.ptr(pose_e), _lib.ptr(pose_g),
                                                _lib.ptr(Ks), _lib.ptr(g), P, max_syms, _lib.ptr(mssd), _lib.ptr(mspd),
                                                _lib.current_stream()), "gdrn_sym_max_dist")
    return mssd, mspd


def ad(models, obj_ids, R_est, t_est, R_gt, t_gt, use_adi, gate=None):
    """ADD (use_adi False) or ADI (True) per pair, mm; gate [P] (False = spheres do not overlap -> inf).  Returns [P]."""
    dev = models.device
    slots = models.slots(obj_ids)
    P = len(slots)
    if P == 0:
        return torch.empty(0, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        po = torch.tensor(slots, dtype=torch.int32, device=dev)
        pose_e, pose_g = _poses(R_est, t_est, P, dev, "ad est"), _poses(R_gt, t_gt, P, dev, "ad gt")
        adi = _vec(use_adi, P, torch.uint8, dev, "ad use_adi")
        g = _gate(gate, P, dev, "ad gate")
        max_pts = max(models.n_pts[s] for s in set(slots))
        L = _lib.lib()
        ws = torch.empty((L.gdrn_ad_workspace_bytes(P, max_pts) + 7) // 8, dtype=torch.float64, device=dev)
        err = torch.empty(P, dtype=torch.float64, device=dev)
        _lib.check(L.gdrn_ad_errors(_lib.ptr(models.pts), _lib.ptr(models.pt_offsets), _lib.ptr(po), _lib.ptr(pose_e),
                                    _lib.ptr(pose_g), _lib.ptr(adi), _lib.ptr(g), P, max_pts, _lib.ptr(ws), ws.numel() * 8,
                                    _lib.ptr(err), _lib.current_stream()), "gdrn_ad_errors")
    return err


def _sym_inputs(models, obj_ids, R_est, t_est, R_gt, t_gt, use_syms, what):
    """(P, pair slots, est / GT poses [P,3,4], use_syms [P] u8, max symmetries of one pair) on the models' device."""
    for x in (models.pts, models.syms, R_est, t_est, R_gt, t_gt, use_syms):
        if torch.is_tensor(x) and not x.is_cuda:
            raise GdrnError(f"{what}: needs CUDA tensors or arrays (no CPU fallback)")
    dev = models.device
    slots = models.slots(obj_ids)
    P = len(slots)
    if P == 0:
        return 0, None, None, None, None, 0
    po = torch.tensor(slots, dtype=torch.int32, device=dev)
    pose_e, pose_g = _poses(R_est, t_est, P, dev, what + " est"), _poses(R_gt, t_gt, P, dev, what + " gt")
    us = _vec(use_syms, P, torch.uint8, dev, what + " use_syms", broadcast=True)
    max_syms = max(models.n_syms[s] if u else 1 for s, u in zip(slots, us.cpu().tolist()))
    return P, po, pose_e, pose_g, us, max_syms


def rt_errors(models, obj_ids, R_est, t_est, R_gt, t_gt, use_syms):
    """Rotation error (deg) and translation error (units of t, mm) of P pairs, pose_error.re / te (use_syms False: the
    GT pose itself) or re_sym / te_sym (True: min over the object's symmetry set, each error on its own).  use_syms is
    one flag or [P].  Returns (re_deg [P], te [P]) f64 CUDA tensors."""
    dev = models.device
    P, po, pose_e, pose_g, us, _ = _sym_inputs(models, obj_ids, R_est, t_est, R_gt, t_gt, use_syms, "rt_errors")
    with torch.cuda.device(dev):
        re_deg = torch.empty(P, dtype=torch.float64, device=dev)
        te = torch.empty(P, dtype=torch.float64, device=dev)
        if P:
            _lib.check(_lib.lib().gdrn_sym_rt_errors(_lib.ptr(models.syms), _lib.ptr(models.sym_offsets), _lib.ptr(po),
                                                     _lib.ptr(pose_e), _lib.ptr(pose_g), _lib.ptr(us), P, _lib.ptr(re_deg),
                                                     _lib.ptr(te), _lib.current_stream()), "gdrn_sym_rt_errors")
    return re_deg, te


def proj_errors(models, obj_ids, R_est, t_est, R_gt, t_gt, K, use_syms):
    """Mean 2D projection distance (px) of P pairs, pose_error.arp_2d (use_syms False) or arp_2d_sym (True: min over the
    object's symmetry set).  K [P,3,3] or [3,3]; use_syms one flag or [P].  Returns [P] f64."""
    dev = models.device
    if torch.is_tensor(K) and not K.is_cuda:
        raise GdrnError("proj_errors: needs CUDA tensors or arrays (no CPU fallback)")
    P, po, pose_e, pose_g, us, max_syms = _sym_inputs(models, obj_ids, R_est, t_est, R_gt, t_gt, use_syms, "proj_errors")
    Ks = _mats(K, P, (3, 3), dev, "proj_errors K") if P else None
    with torch.cuda.device(dev):
        err = torch.empty(P, dtype=torch.float64, device=dev)
        if P:
            _lib.check(_lib.lib().gdrn_sym_proj_mean(_lib.ptr(models.pts), _lib.ptr(models.pt_offsets),
                                                     _lib.ptr(models.syms), _lib.ptr(models.sym_offsets), _lib.ptr(po),
                                                     _lib.ptr(pose_e), _lib.ptr(pose_g), _lib.ptr(Ks), _lib.ptr(us), P,
                                                     max_syms, _lib.ptr(err), _lib.current_stream()), "gdrn_sym_proj_mean")
    return err


# ---------------------------------------------------------------------------------------------------------------------
# Rendering for VSD: each estimate and each GT instance rendered once (float z, the egl renderer type's near / far)
VSD_ZNEAR, VSD_ZFAR = 0.01, 10000.0


class VsdMeshes:
    """The meshes of a dataset (mm), each uploaded once to the rasteriser's registry as a renderer.Model3D; ids maps
    obj_id to its registry id.  meshes: {obj_id: (verts [V,3], faces [F,3])} or {obj_id: (verts, faces, colors [V,3]
    in [0,1] or None)}, optionally followed by uvs [V,2] and texture [h,w,3] u8 (row 0 at t = 0), as arrays or CPU
    tensors."""

    def __init__(self, meshes, device="cuda"):
        from .renderer import Model3D

        self.device = torch.device(device)
        self.ids = {int(o): Model3D(m[0], m[1], device=self.device, colors=m[2] if len(m) > 2 else None,
                                    uvs=m[3] if len(m) > 3 else None, texture=m[4] if len(m) > 4 else None).mesh_id
                    for o, m in meshes.items()}

    def render(self, obj_ids, R, t, K, H, W):
        """Float-z depth [n,H,W] of obj_ids[i] at pose (R[i], t[i]) with intrinsics K[i] (mm)."""
        from . import renderer

        n = len(obj_ids)
        try:
            ids = torch.tensor([self.ids[int(o)] for o in obj_ids], dtype=torch.int32, device=self.device)
        except KeyError as e:
            raise GdrnError(f"VsdMeshes: no mesh for obj_id {e.args[0]}") from None
        poses = torch.from_numpy(np.concatenate([np.asarray(R, np.float64).reshape(n, 3, 3),
                                                 np.asarray(t, np.float64).reshape(n, 3, 1)], axis=2)).to(self.device)
        Ks = torch.from_numpy(np.asarray(K, np.float64).reshape(n, 3, 3)).to(self.device)
        return renderer.render_meshes(ids, poses, Ks, H, W, VSD_ZNEAR, VSD_ZFAR, quantize_bits=0)


# ---------------------------------------------------------------------------------------------------------------------
# eval_calc_errors.py:255-480: the error loop, one GPU call per error type and chunk of images
ERROR_TYPES = ("vsd", "mssd", "mspd", "ad", "add", "adi")
VSD_DELTAS = {"hb": 15, "hbs": 15, "icbin": 15, "icmi": 15, "itodd": 5, "lm": 15, "lmo": 15, "ruapc": 15, "tless": 15,
              "tudl": 15, "tyol": 15, "ycbv": 15, "hope": 15}
VSD_TAUS = list(np.arange(0.05, 0.51, 0.05))


def select_estimates(ests, targets, n_top=-1, skip_missing=True):
    """Targets organised by scene / image / object, each with its estimates sorted by score (stable, descending) and cut
    to n_top (0 = all, -1 = the target's inst_count).  -> [(scene_id, im_id, obj_id, [(est_id, est), ...])]."""
    targets_org = {}
    for tg in targets:
        targets_org.setdefault(tg["scene_id"], {}).setdefault(tg["im_id"], {})[tg["obj_id"]] = tg
    ests_org = {}
    for e in ests:
        ests_org.setdefault(e["scene_id"], {}).setdefault(e["im_id"], {}).setdefault(e["obj_id"], []).append(e)
    out = []
    for scene_id, scene_targets in targets_org.items():
        for im_id, im_targets in scene_targets.items():
            for obj_id, tg in im_targets.items():
                n_top_curr = None if n_top == 0 else (tg["inst_count"] if n_top == -1 else n_top)
                obj_ests = ests_org.get(scene_id, {}).get(im_id, {}).get(obj_id, [])
                if not skip_missing and len(obj_ests) < n_top_curr:
                    raise ValueError(f"Not enough estimates for scene: {scene_id}, im: {im_id}, obj: {obj_id} "
                                     f"(provided: {len(obj_ests)}, expected: {n_top_curr})")
                srt = sorted(enumerate(obj_ests), key=lambda x: x[1]["score"], reverse=True)
                out.append((scene_id, im_id, obj_id, srt[slice(0, n_top_curr)]))
    return out


def calc_errors(error_type, dataset, ests, targets, scene_gts, scene_cameras, models_info, models=None, meshes=None,
                load_depth=None, n_top=-1, skip_missing=True, vsd_delta=None, vsd_taus=None, vsd_normalized_by_diameter=True,
                max_bytes=2 << 30):
    """Errors of every selected estimate w.r.t. every GT instance of its object, as eval_calc_errors.py computes them.

    scene_gts / scene_cameras: {scene_id: load_scene_gt / load_scene_camera output}; models: PoseErrorModels (mssd, mspd,
    ad*); meshes: VsdMeshes and load_depth(scene_id, im_id) -> [H,W] f32 test depth in mm (vsd).  The pairs of a chunk of
    images go in one call; chunks hold at most max_bytes of VSD renders and counters, which changes no output bit.
    -> {scene_id: [{im_id, obj_id, est_id, score, errors: {gt_id: [e, ...]}}]} in the reference's order."""
    if error_type not in ERROR_TYPES:
        raise ValueError(f"error type {error_type!r} is not supported (supported: {', '.join(ERROR_TYPES)})")
    records, pairs, arrays = error_pairs(ests, targets, scene_gts, scene_cameras, models_info, n_top, skip_missing)
    if not pairs:
        return records
    diam, R_e, t_e, R_g, t_g, K, obj = arrays
    if error_type == "vsd":
        errs = _calc_vsd(pairs, obj, R_e, t_e, R_g, t_g, K, diam, meshes, load_depth, vsd_delta,
                         VSD_TAUS if vsd_taus is None else vsd_taus, vsd_normalized_by_diameter, max_bytes)
    else:
        gate = np.array([spheres_overlap(t_e[i], t_g[i], diam[i]) for i in range(len(pairs))])
        if error_type in ("mssd", "mspd"):
            mssd, mspd = mssd_mspd(models, obj, R_e, t_e, R_g, t_g, K, gate_mssd=gate)
            e = (mssd if error_type == "mssd" else mspd).cpu().numpy()
        else:
            use_adi = [error_type == "adi" or (error_type == "ad" and is_symmetric(dataset, o, models_info[o])) for o in obj]
            e = ad(models, obj, R_e, t_e, R_g, t_g, use_adi, gate=gate).cpu().numpy()
        errs = e[:, None]
    return fill_errors(records, pairs, errs)


def error_pairs(ests, targets, scene_gts, scene_cameras, models_info, n_top=-1, skip_missing=True):
    """The (estimate, GT) pairs of eval_calc_errors.py's loop: every selected estimate with every GT instance of its
    object.  -> (records {scene_id: [{im_id, obj_id, est_id, score, errors: {}}]}, pairs [(record, gt_id, scene_id,
    im_id, obj_id, est, gt)], (diameters [P], R_e [P,3,3], t_e [P,3], R_g, t_g, K [P,3,3], obj_ids [P])) -- the
    arrays are None when there is no pair."""
    records, pairs = {}, []
    for scene_id, im_id, obj_id, srt in select_estimates(ests, targets, n_top, skip_missing):
        scene_errs = records.setdefault(scene_id, [])
        for est_id, est in srt:
            rec = {"im_id": im_id, "obj_id": obj_id, "est_id": est_id, "score": est["score"], "errors": {}}
            scene_errs.append(rec)
            for gt_id, gt in enumerate(scene_gts[scene_id][im_id]):
                if gt["obj_id"] == obj_id:
                    pairs.append((rec, gt_id, scene_id, im_id, obj_id, est, gt))
    if not pairs:
        return records, pairs, None
    diam = np.array([float(models_info[p[4]]["diameter"]) for p in pairs])
    R_e = np.stack([np.asarray(p[5]["R"], np.float64).reshape(3, 3) for p in pairs])
    t_e = np.stack([np.asarray(p[5]["t"], np.float64).reshape(3) for p in pairs])
    R_g = np.stack([np.asarray(p[6]["cam_R_m2c"], np.float64).reshape(3, 3) for p in pairs])
    t_g = np.stack([np.asarray(p[6]["cam_t_m2c"], np.float64).reshape(3) for p in pairs])
    K = np.stack([np.asarray(scene_cameras[p[2]][p[3]]["cam_K"], np.float64).reshape(3, 3) for p in pairs])
    return records, pairs, (diam, R_e, t_e, R_g, t_g, K, [p[4] for p in pairs])


def fill_errors(records, pairs, errs):
    """Store row p of errs [P, n] as the error list of pair p in its record.  -> records."""
    for p, e in zip(pairs, errs):
        p[0]["errors"][p[1]] = [float(v) for v in e]
    return records


def _calc_vsd(pairs, obj, R_e, t_e, R_g, t_g, K, diam, meshes, load_depth, delta, taus, normalized, max_bytes):
    gate = np.array([sphere_projections_overlap(0.5 * diam[i], t_e[i], t_g[i]) for i in range(len(pairs))])
    images = list(dict.fromkeys((p[2], p[3]) for p in pairs))   # in first-use order
    out = np.ones((len(pairs), len(taus)))
    dev = meshes.device
    chunk, chunk_bytes, HW = [], 0, None

    def flush(chunk):
        im_index = {im: k for k, im in enumerate(chunk)}
        sel = [i for i, p in enumerate(pairs) if (p[2], p[3]) in im_index and gate[i]]
        if not sel:
            return
        tests = [np.asarray(load_depth(*im), np.float32) for im in chunk]
        H, W = tests[0].shape
        est_key, gt_key = {}, {}   # one render per estimate record and per GT instance
        for i in sel:
            est_key.setdefault(id(pairs[i][0]), i)
            gt_key.setdefault((pairs[i][2], pairs[i][3], pairs[i][1]), i)
        ei, gi = list(est_key.values()), list(gt_key.values())
        with torch.cuda.device(dev):
            d_est = meshes.render([obj[i] for i in ei], R_e[ei], t_e[ei], K[ei], H, W)
            d_gt = meshes.render([obj[i] for i in gi], R_g[gi], t_g[gi], K[gi], H, W)
            d_test = torch.from_numpy(np.stack(tests)).to(dev)
            pe = [ei.index(est_key[id(pairs[i][0])]) for i in sel]
            pg = [gi.index(gt_key[(pairs[i][2], pairs[i][3], pairs[i][1])]) for i in sel]
            pim = [im_index[(pairs[i][2], pairs[i][3])] for i in sel]
            e = vsd(d_est, d_gt, d_test, pe, pg, pim, K[sel], diam[sel], taus, delta, normalized).cpu().numpy()
        out[sel] = e

    for im in images:
        n_im = sum(1 for p in pairs if (p[2], p[3]) == im)
        if HW is None:
            HW = int(np.asarray(load_depth(*im)).size)
        im_bytes = HW * 4 * (1 + 2 * n_im) + HW * 8 * n_im + n_im * (len(taus) + 2) * 8   # test + renders + scratch
        if chunk and chunk_bytes + im_bytes > max_bytes:
            flush(chunk)
            chunk, chunk_bytes = [], 0
        chunk.append(im)
        chunk_bytes += im_bytes
    if chunk:
        flush(chunk)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Scores (host): eval_calc_scores.py:166-297, pose_matching.py, score.py -- cheap, and restated exactly
CORRECT_TH = {
    "vsd": [[th] for th in np.arange(0.05, 0.51, 0.05)],
    "mssd": [[th] for th in np.arange(0.05, 0.51, 0.05)],
    "mspd": [[th] for th in np.arange(5, 51, 5)],
    "ad": [[th] for th in [0.02, 0.05, 0.1]],
    "add": [[th] for th in [0.02, 0.05, 0.1]],
    "adi": [[th] for th in [0.02, 0.05, 0.1]],
}
NORMALIZED_BY_DIAMETER = ("ad", "add", "adi", "mssd")
NORMALIZED_BY_IM_WIDTH = ("mspd",)


def get_error_signature(error_type, n_top, **kwargs):
    """misc.get_error_signature (misc.py:1244-1260)."""
    error_sign = "error:" + error_type + "_ntop:" + str(n_top)
    if error_type == "vsd":
        tau = "inf" if kwargs["vsd_tau"] == float("inf") else "{:.3f}".format(kwargs["vsd_tau"])
        error_sign += "_delta:{:.3f}_tau:{}".format(kwargs["vsd_delta"], tau)
    return error_sign


def get_score_signature(correct_th, visib_gt_min):
    """misc.get_score_signature (misc.py:1263-1271)."""
    return "th:" + "-".join(["{:.3f}".format(t) for t in correct_th]) + "_min-visib:{:.3f}".format(visib_gt_min)


def match_poses(errs, error_ths, max_ests_count=0, gt_valid_mask=None):
    """pose_matching.match_poses: greedy, in the order of decreasing score."""
    errs_sorted = sorted(errs, key=lambda e: e["score"], reverse=True)
    if max_ests_count > 0:
        errs_sorted = errs_sorted[:max_ests_count]
    n = len(list(error_ths))
    matches, gt_matched = [], []
    for e in errs_sorted:
        best_gt_id, best_error = -1, list(error_ths)
        for gt_id, error in e["errors"].items():
            is_valid = not gt_valid_mask or gt_valid_mask[gt_id]
            if is_valid and gt_id not in gt_matched:
                if np.all([error[i] < best_error[i] for i in range(n)]):
                    best_gt_id, best_error = gt_id, error
        if best_gt_id >= 0:
            gt_matched.append(best_gt_id)
            matches.append({"est_id": e["est_id"], "gt_id": best_gt_id, "score": e["score"], "error": best_error,
                            "error_norm": [best_error[i] / float(error_ths[i]) for i in range(n)]})
    return matches


def match_poses_scene(scene_id, scene_gt, scene_gt_valid, scene_errs, correct_th, n_top):
    """pose_matching.match_poses_scene: one match record per GT instance."""
    org = {}
    for e in scene_errs:
        org.setdefault(e["im_id"], {}).setdefault(e["obj_id"], []).append(e)
    scene_matches = []
    for im_id, im_gts in scene_gt.items():
        im_matches = [{"scene_id": scene_id, "im_id": im_id, "obj_id": gt["obj_id"], "gt_id": gt_id, "est_id": -1,
                       "score": -1, "error": -1, "error_norm": -1, "valid": scene_gt_valid[im_id][gt_id]}
                      for gt_id, gt in enumerate(im_gts)]
        for obj_id in set(gt["obj_id"] for gt in im_gts):
            if im_id in org and obj_id in org[im_id]:
                for m in match_poses(org[im_id][obj_id], correct_th, n_top, scene_gt_valid[im_id]):
                    g = im_matches[m["gt_id"]]
                    g["est_id"], g["score"], g["error"], g["error_norm"] = m["est_id"], m["score"], m["error"], m["error_norm"]
        scene_matches += im_matches
    return scene_matches


def calc_recall(tp_count, targets_count):
    return 0.0 if targets_count == 0 else tp_count / float(targets_count)


def calc_localization_scores(scene_ids, obj_ids, matches, n_top):
    """score.calc_localization_scores (without the printing)."""
    insts = {i: {j: {} for j in scene_ids} for i in obj_ids}
    for m in matches:
        if m["valid"]:
            d = insts[m["obj_id"]][m["scene_id"]]
            d[m["im_id"]] = d.get(m["im_id"], 0) + 1
    tars, obj_tars, scene_tars = 0, {i: 0 for i in obj_ids}, {i: 0 for i in scene_ids}
    for obj_id, obj_insts in insts.items():
        for scene_id, scene_insts in obj_insts.items():
            count = sum(np.minimum(n_top, list(scene_insts.values()))) if n_top > 0 else sum(list(scene_insts.values()))
            tars += count
            obj_tars[obj_id] += count
            scene_tars[scene_id] += count
    tps, obj_tps, scene_tps = 0, {i: 0 for i in obj_ids}, {i: 0 for i in scene_ids}
    for m in matches:
        if m["valid"] and m["est_id"] != -1:
            tps += 1
            obj_tps[m["obj_id"]] += 1
            scene_tps[m["scene_id"]] += 1
    obj_recalls = {i: calc_recall(obj_tps[i], obj_tars[i]) for i in obj_ids}
    scene_recalls = {i: float(calc_recall(scene_tps[i], scene_tars[i])) for i in scene_ids}
    return {"recall": float(calc_recall(tps, tars)), "obj_recalls": obj_recalls,
            "mean_obj_recall": float(np.mean(list(obj_recalls.values())).squeeze()), "scene_recalls": scene_recalls,
            "mean_scene_recall": float(np.mean(list(scene_recalls.values())).squeeze()), "gt_count": len(matches),
            "targets_count": int(tars), "tp_count": int(tps)}


def gt_valid_masks(scene_targets, scene_gt, scene_gt_info, visib_gt_min=-1):
    """eval_calc_scores.py:199-233: which GT instances count, per image of one scene."""
    scene_gt_curr, valid = {}, {}
    for im_id, im_targets in scene_targets.items():
        scene_gt_curr[im_id] = im_gt = scene_gt[im_id]
        im_gt_info = scene_gt_info[im_id]
        valid[im_id] = [True] * len(im_gt)
        if visib_gt_min >= 0:
            for gt_id, gt in enumerate(im_gt):
                valid[im_id][gt_id] = gt["obj_id"] in im_targets and im_gt_info[gt_id]["visib_fract"] >= visib_gt_min
        else:
            order = sorted(range(len(im_gt)), key=lambda g: im_gt_info[g]["visib_fract"], reverse=True)
            to_add = {o: tg["inst_count"] for o, tg in im_targets.items()}
            for gt_id in order:
                o = im_gt[gt_id]["obj_id"]
                if o in to_add and to_add[o] > 0:
                    valid[im_id][gt_id] = True
                    to_add[o] -= 1
                else:
                    valid[im_id][gt_id] = False
    return scene_gt_curr, valid


def calc_scores(error_type, scene_errs, targets, scene_gts, scene_gt_infos, models_info, im_width, correct_th, n_top,
                scene_ids=None, obj_ids=None, visib_gt_min=-1):
    """eval_calc_scores.py for one error directory: normalise (by diameter or by 640 / image width), match per scene,
    score.  scene_errs: {scene_id: records with ONE error value per GT} (for VSD: one tau).  -> (scores, matches)."""
    targets_org = {}
    for tg in targets:
        targets_org.setdefault(tg["scene_id"], {}).setdefault(tg["im_id"], {})[tg["obj_id"]] = tg
    matches = []
    for scene_id, scene_targets in targets_org.items():
        gt_curr, valid = gt_valid_masks(scene_targets, scene_gts[scene_id], scene_gt_infos[scene_id], visib_gt_min)
        errs = [{**e, "errors": {g: list(v) for g, v in e["errors"].items()}} for e in scene_errs.get(scene_id, [])]
        if error_type in NORMALIZED_BY_DIAMETER:
            for err in errs:
                diameter = float(models_info[err["obj_id"]]["diameter"])
                for g in err["errors"]:
                    err["errors"][g] = [e / diameter for e in err["errors"][g]]
        if error_type in NORMALIZED_BY_IM_WIDTH:
            factor = 640.0 / float(im_width)
            for err in errs:
                for g in err["errors"]:
                    err["errors"][g] = [factor * e for e in err["errors"][g]]
        matches += match_poses_scene(scene_id, gt_curr, valid, errs, correct_th, n_top)
    scene_ids = sorted(targets_org) if scene_ids is None else scene_ids
    obj_ids = sorted(models_info) if obj_ids is None else obj_ids
    return calc_localization_scores(scene_ids, obj_ids, matches, n_top), matches


def split_errors_per_tau(scene_errs, n_taus):
    """eval_calc_errors.py:620-633: the VSD records of one tau each."""
    return [{s: [{**e, "errors": {g: [v[k]] for g, v in e["errors"].items()}} for e in recs] for s, recs in scene_errs.items()}
            for k in range(n_taus)]


def average_recalls(error_type, errors, targets, scene_gts, scene_gt_infos, models_info, im_width, n_top=-1,
                    scene_ids=None, obj_ids=None, visib_gt_min=-1, n_taus=len(VSD_TAUS), correct_th=CORRECT_TH):
    """eval_pose_results_more.py:327-360: the recall at every threshold of correct_th[error_type] (and, for VSD, every
    tau) and their mean.  errors: calc_errors output.  -> (average recall, [(sign index, threshold, scores, matches)])."""
    per_sign = split_errors_per_tau(errors, n_taus) if error_type == "vsd" else [errors]
    details = []
    for si, errs in enumerate(per_sign):
        for th in correct_th[error_type]:
            scores, matches = calc_scores(error_type, errs, targets, scene_gts, scene_gt_infos, models_info, im_width, th,
                                          n_top, scene_ids, obj_ids, visib_gt_min)
            details.append((si, th, scores, matches))
    return np.mean([d[2]["recall"] for d in details]), details


def evaluate(error_types, dataset, ests, targets, scene_gts, scene_cameras, scene_gt_infos, models_info, im_width,
             models=None, meshes=None, load_depth=None, n_top=-1, max_bytes=2 << 30, scene_ids=None, obj_ids=None,
             calc=calc_errors, correct_th=CORRECT_TH):
    """The BOP19 average recalls of eval_pose_results_more.py:250-380 for the given error types, computed in memory.
    calc / correct_th: the error dispatch (calc_errors' signature) and the thresholds per error type.
    -> ({'bop19_average_recall_<type>': AR, ..., 'bop19_average_recall': mean of vsd / mssd / mspd}, {type: errors})."""
    final, all_errors = {}, {}
    for et in error_types:
        errs = calc(et, dataset, ests, targets, scene_gts, scene_cameras, models_info, models, meshes, load_depth,
                           n_top, True, VSD_DELTAS.get(dataset, 15), VSD_TAUS, True, max_bytes)
        all_errors[et] = errs
        final["bop19_average_recall_" + et] = average_recalls(et, errs, targets, scene_gts, scene_gt_infos, models_info,
                                                              im_width, n_top, scene_ids, obj_ids,
                                                              correct_th=correct_th)[0]
    if all(t in error_types for t in ("mspd", "mssd", "vsd")):
        final["bop19_average_recall"] = np.mean([final["bop19_average_recall_" + t] for t in ("mspd", "mssd", "vsd")])
    return final, all_errors


# ---------------------------------------------------------------------------------------------------------------------
# BOP file I/O (lib/pysixd/inout.py, docs/bop_datasets_format.md), kept to what the evaluation reads and writes
IM_SIZES = {"tless": (720, 540), "itodd": (1280, 960), "hope": (1920, 1080)}   # (width, height); the others 640 x 480


def load_json(path, keys_to_int=False):
    def conv(x):
        return {int(k) if k.lstrip("-").isdigit() else k: v for k, v in x}

    with open(path, "r") as f:
        return json.load(f, object_pairs_hook=conv) if keys_to_int else json.load(f)


def save_json(path, content, sort=False):
    """inout.save_json's layout: one top-level element per line."""
    with open(path, "w") as f:
        if isinstance(content, dict):
            items = sorted(content.items(), key=lambda x: x[0]) if sort else list(content.items())
            f.write("{\n" + ",\n".join('  "{}": {}'.format(k, json.dumps(v, sort_keys=True)) for k, v in items) + "\n}")
        elif isinstance(content, list):
            f.write("[\n" + ",\n".join("  {}".format(json.dumps(e, sort_keys=True)) for e in content) + "\n]")
        else:
            json.dump(content, f, sort_keys=True)


def load_scene_gt(path):
    scene_gt = load_json(path, keys_to_int=True)
    for im_gt in scene_gt.values():
        for gt in im_gt:
            gt["cam_R_m2c"] = np.array(gt["cam_R_m2c"], np.float64).reshape((3, 3))
            gt["cam_t_m2c"] = np.array(gt["cam_t_m2c"], np.float64).reshape((3, 1))
    return scene_gt


def load_scene_camera(path):
    cams = load_json(path, keys_to_int=True)
    for cam in cams.values():
        cam["cam_K"] = np.array(cam["cam_K"], np.float64).reshape((3, 3))
    return cams


def load_depth(path, depth_scale=1.0):
    """Depth image (PNG / TIF) as f32, times depth_scale in f32 as the reference scales it in place (-> mm)."""
    import cv2

    d = cv2.imread(path, cv2.IMREAD_ANYDEPTH)
    if d is None:
        raise FileNotFoundError(path)
    d = d.astype(np.float32)
    d *= np.float32(depth_scale)
    return d


def load_bop_results(path):
    """inout.load_bop_results, bop19 format: scene_id,im_id,obj_id,score,R,t,time (R row-major, t in mm)."""
    results = []
    with open(path, "r") as f:
        for line_id, line in enumerate(f):
            if line_id == 0 and "scene_id,im_id,obj_id,score,R,t,time" in line:
                continue
            elems = line.split(",")
            if len(elems) != 7:
                raise ValueError("A line does not have 7 comma-sep. elements: {}".format(line))
            results.append({"scene_id": int(elems[0]), "im_id": int(elems[1]), "obj_id": int(elems[2]),
                            "score": float(elems[3]),
                            "R": np.array(list(map(float, elems[4].split())), np.float64).reshape((3, 3)),
                            "t": np.array(list(map(float, elems[5].split())), np.float64).reshape((3, 1)),
                            "time": float(elems[6])})
    return results


def write_bop_results_csv(records, path):
    """Results CSV as save_and_eval_results writes it, from GdrnPredictor records {scene_id, im_id, obj_id, score,
    R [3,3], t [3] in metres, time}: t is written in mm (x 1000), as pose_prediction_to_json does."""
    with open(path, "w") as f:
        f.write("scene_id,im_id,obj_id,score,R,t,time\n")
        for r in records:
            R = np.asarray(r["R"], np.float64).reshape(-1).tolist()
            t = (np.asarray(r["t"], np.float64).reshape(-1) * 1000).tolist()
            f.write(",".join([str(int(r["scene_id"])), str(int(r["im_id"])), str(int(r["obj_id"])), "{}".format(r["score"]),
                              " ".join("{}".format(e) for e in R), " ".join("{}".format(e) for e in t),
                              "{}".format(r.get("time", -1))]) + "\n")


class BopSplit:
    """Paths and per-scene data of one dataset split in the standard BOP layout."""

    def __init__(self, datasets_path, dataset, split, split_type=None):
        self.dataset = dataset
        self.base_path = os.path.join(datasets_path, dataset)
        self.split_path = os.path.join(self.base_path, split + ("_" + split_type if split_type else ""))
        self.models_path = os.path.join(self.base_path, "models_eval")
        self.im_size = IM_SIZES.get(dataset, (640, 480))
        self.scene_ids = sorted(int(d) for d in os.listdir(self.split_path)
                                if d.isdigit() and os.path.isdir(os.path.join(self.split_path, d)))

    def scene_file(self, scene_id, name):
        return os.path.join(self.split_path, "{:06d}".format(scene_id), name)

    def models_info(self):
        return load_json(os.path.join(self.models_path, "models_info.json"), keys_to_int=True)

    def model(self, obj_id):
        from .ply import load_ply

        return load_ply(os.path.join(self.models_path, "obj_{:06d}.ply".format(obj_id)))

    def depth(self, scene_id, im_id, depth_scale):
        for ext in (".png", ".tif"):
            path = self.scene_file(scene_id, os.path.join("depth", "{:06d}{}".format(im_id, ext)))
            if os.path.exists(path):
                return load_depth(path, depth_scale)
        raise FileNotFoundError(self.scene_file(scene_id, os.path.join("depth", "{:06d}.png".format(im_id))))


# ---------------------------------------------------------------------------------------------------------------------
# Command line: the arguments save_and_eval_results passes to VAL.SCRIPT_PATH, the files of eval_pose_results_more.py
def parse_args(argv=None):
    return parse_eval_args(argv, "BOP19 pose-error evaluation on the GPU (VSD, MSSD, MSPD, AD / ADD / ADI)", "mspd,mssd,vsd",
                           ERROR_TYPES)


def parse_eval_args(argv, description, default_error_types, known_error_types):
    """The command line of an evaluation script; error types outside known_error_types are rejected with a message."""
    ap = argparse.ArgumentParser(description=description)
    ap.add_argument("--results_path", default="output/bop_results")
    ap.add_argument("--result_filenames", required=True, help="comma-separated result CSV names")
    ap.add_argument("--renderer_type", default="cuda", help="accepted for compatibility; renders always use the CUDA rasteriser")
    ap.add_argument("--error_types", default=default_error_types)
    ap.add_argument("--eval_path", default="output/bop_eval/")
    ap.add_argument("--targets_filename", default="test_targets_bop19.json")
    ap.add_argument("--n_top", default=-1, type=int)
    ap.add_argument("--score_only", action="store_true", help="read errors written earlier instead of computing them")
    ap.add_argument("--datasets_path", default=os.environ.get("BOP_PATH", "datasets/BOP_DATASETS/"))
    ap.add_argument("--dataset", default=None)
    ap.add_argument("--max_bytes", default=2 << 30, type=int, help="device memory budget of one VSD chunk")
    args = ap.parse_args(argv)
    args.result_filenames = args.result_filenames.split(",")
    args.error_types = args.error_types.split(",")
    bad = [t for t in args.error_types if t not in known_error_types]
    if bad:
        ap.error("error types {} are not supported here (supported: {})".format(",".join(bad), ",".join(known_error_types)))
    return args


def run(args, calc=calc_errors, correct_th=CORRECT_TH):
    """Evaluate every result file; writes errors_*.json, scores_*.json, matches_*.json and scores_bop19.json under
    eval_path/<result name>/ with the reference's signatures.  calc / correct_th: the error dispatch and thresholds, as
    for evaluate.  -> {result name: final scores}."""
    out = {}
    for result_filename in args.result_filenames:
        t0 = time.time()
        result_name = os.path.splitext(os.path.basename(result_filename))[0]
        info = result_name.split("_")[1].split("-")
        dataset = args.dataset or info[0]
        ds = BopSplit(args.datasets_path, info[0], info[1], info[2] if len(info) > 2 else None)
        ests = load_bop_results(os.path.join(args.results_path, result_filename))
        times = {}
        for e in ests:
            times.setdefault((e["scene_id"], e["im_id"]), e["time"])
        avg_time = float(np.mean(list(times.values()))) if times and min(times.values()) >= 0 else -1.0
        targets = load_json(os.path.join(ds.base_path, args.targets_filename))
        scene_ids = sorted(set(t["scene_id"] for t in targets))
        scene_gts = {s: load_scene_gt(ds.scene_file(s, "scene_gt.json")) for s in scene_ids}
        scene_cams = {s: load_scene_camera(ds.scene_file(s, "scene_camera.json")) for s in scene_ids}
        scene_infos = {s: load_json(ds.scene_file(s, "scene_gt_info.json"), keys_to_int=True) for s in scene_ids}
        models_info = ds.models_info()
        obj_ids = sorted(models_info)
        models = meshes = None
        if not args.score_only:
            plys = {o: ds.model(o) for o in obj_ids}
            if any(t != "vsd" for t in args.error_types):
                models = PoseErrorModels({o: m["pts"] for o, m in plys.items()}, models_info)
            if "vsd" in args.error_types:
                meshes = VsdMeshes({o: (m["pts"], m["faces"]) for o, m in plys.items()})
        final = {}
        delta = VSD_DELTAS.get(dataset, 15)
        for et in sorted(args.error_types):
            signs = ([get_error_signature(et, args.n_top, vsd_delta=delta, vsd_tau=tau) for tau in VSD_TAUS] if et == "vsd"
                     else [get_error_signature(et, args.n_top)])
            if args.score_only:
                per_sign = [{s: load_json(os.path.join(args.eval_path, result_name, sg, "errors_{:06d}.json".format(s)),
                                          keys_to_int=True) for s in scene_ids} for sg in signs]
            else:
                errs = calc(et, dataset, ests, targets, scene_gts, scene_cams, models_info, models, meshes,
                                   lambda s, i: ds.depth(s, i, scene_cams[s][i].get("depth_scale", 1.0)), args.n_top, True,
                                   delta, VSD_TAUS, True, args.max_bytes)
                per_sign = split_errors_per_tau(errs, len(VSD_TAUS)) if et == "vsd" else [errs]
                for sg, e in zip(signs, per_sign):
                    d = os.path.join(args.eval_path, result_name, sg)
                    os.makedirs(d, exist_ok=True)
                    for s in scene_ids:
                        save_json(os.path.join(d, "errors_{:06d}.json".format(s)), e.get(s, []))
            recalls = []
            for sg, e in zip(signs, per_sign):
                for th in correct_th[et]:
                    scores, matches = calc_scores(et, e, targets, scene_gts, scene_infos, models_info, ds.im_size[0], th,
                                                  args.n_top, ds.scene_ids, obj_ids)
                    d = os.path.join(args.eval_path, result_name, sg)
                    os.makedirs(d, exist_ok=True)
                    ssign = get_score_signature(th, -1)
                    save_json(os.path.join(d, "scores_{}.json".format(ssign)), scores)
                    save_json(os.path.join(d, "matches_{}.json".format(ssign)), matches)
                    recalls.append(scores["recall"])
            final["bop19_average_recall_" + et] = np.mean(recalls)
        if all(t in args.error_types for t in ("mspd", "mssd", "vsd")):
            final["bop19_average_recall"] = np.mean([final["bop19_average_recall_" + t] for t in ("mspd", "mssd", "vsd")])
        final["bop19_average_time_per_image"] = avg_time
        os.makedirs(os.path.join(args.eval_path, result_name), exist_ok=True)
        save_json(os.path.join(args.eval_path, result_name, "scores_bop19.json"), {k: float(v) for k, v in final.items()},
                  sort=True)
        print("{}: {} ({:.1f} s)".format(result_name, json.dumps({k: float(v) for k, v in sorted(final.items())}),
                                         time.time() - t0))
        out[result_name] = final
    return out


if __name__ == "__main__":
    run(parse_args())
