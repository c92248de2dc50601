"""Python surfaces of the reference's native extensions, backed by libgdrn_b200.so.

Mirrors (same names, argument meaning and error behaviour):
  * core/csrc/fps/fps_utils.py:6-21                  -> farthest_point_sampling(pts, sn, init_center)
  * core/csrc/ransac_voting (pybind module)          -> ransac_voting.{generate_hypothesis, voting_for_hypothesis,
        generate_hypothesis_vanishing_point, voting_for_hypothesis_vanishing_point}
    and the driver core/csrc/ransac_voting/ransac_voting_gpu.py:7-330 -> ransac_voting_layer / _v3 /
    estimate_voting_distribution_with_mean, as ONE device-side call (csrc/ransac_layer.cu)
  * core/csrc/torch_nndistance/torch_nndistance.py   -> NNDFunction, nnd
  * core/csrc/flow/flow_torch.py:15-40               -> FlowFunction, flow; flow_cuda.forward
  * core/csrc/uncertainty_pnp/un_pnp_utils.py:11-78  -> uncertainty_pnp (EPnP init stays cv2 on the host)
There is no CPU fallback: CUDA tensors in, CUDA tensors out (the numpy FPS entry stages through the GPU).
"""
import ctypes

import numpy as np
import torch
from torch.autograd import Function

from . import _lib


def _check_cuda_contig(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")


# ------------------------------------------------------------------------------------------------- FPS
def farthest_point_sampling(pts, sn, init_center=False):
    """numpy [pn,3] -> pts[idxs] (fps_utils.py:6-21)."""
    pn, _ = pts.shape
    assert pts.shape[1] == 3
    pts = np.ascontiguousarray(pts, np.float32)
    idxs = np.ascontiguousarray(np.zeros([sn], np.int32))
    L = _lib.lib()
    fn = L.farthest_point_sampling_init_center if init_center else L.farthest_point_sampling
    fn(pts.ctypes.data_as(ctypes.c_void_p), idxs.ctypes.data_as(ctypes.c_void_p), pn, sn)
    return pts[idxs]


@_lib.on_device(0)
def farthest_point_sampling_idx(pts, sn, start_idx=None):
    """Batched device FPS: pts [b,pn,3] f32 CUDA -> idx [b,sn] i32. start_idx None = init_center."""
    _check_cuda_contig(pts, "pts")
    b, pn, _ = pts.shape
    idx = torch.empty((b, sn), dtype=torch.int32, device=pts.device)
    st = None
    if start_idx is not None:
        st = start_idx.to(device=pts.device, dtype=torch.int32).contiguous()
    _lib.check(_lib.lib().gdrn_fps_cuda(_lib.ptr(pts), _lib.ptr(idx), pn, sn, b, _lib.ptr(st), _lib.current_stream()),
               "gdrn_fps_cuda")
    return idx


# --------------------------------------------------------------------------------------- ransac_voting
class _RansacVotingModule:
    """Drop-in for the pybind module `ransac_voting` (ransac_voting.cpp:112-117)."""

    @staticmethod
    def _dims(direct, coords):
        for t, n in ((direct, "direct"), (coords, "coords")):
            _check_cuda_contig(t, n)
        tn, vn, two = direct.shape
        assert two == 2 and tuple(coords.shape) == (tn, 2)
        return tn, vn

    @_lib.on_device(1)
    def generate_hypothesis(self, direct, coords, idxs):
        tn, vn = self._dims(direct, coords)
        _check_cuda_contig(idxs, "idxs")
        hn = idxs.shape[0]
        assert tuple(idxs.shape) == (hn, vn, 2) and idxs.dtype == torch.int32
        hypo = torch.zeros((hn, vn, 2), dtype=direct.dtype, device=direct.device)
        _lib.check(_lib.lib().rv_generate_hypothesis(_lib.ptr(direct), _lib.ptr(coords), _lib.ptr(idxs), _lib.ptr(hypo),
                                                     tn, vn, hn, _lib.current_stream()), "rv_generate_hypothesis")
        return hypo

    @_lib.on_device(1)
    def generate_hypothesis_vanishing_point(self, direct, coords, idxs):
        tn, vn = self._dims(direct, coords)
        _check_cuda_contig(idxs, "idxs")
        hn = idxs.shape[0]
        assert tuple(idxs.shape) == (hn, vn, 2) and idxs.dtype == torch.int32
        hypo = torch.zeros((hn, vn, 3), dtype=direct.dtype, device=direct.device)
        _lib.check(_lib.lib().rv_generate_hypothesis_vanishing_point(
            _lib.ptr(direct), _lib.ptr(coords), _lib.ptr(idxs), _lib.ptr(hypo), tn, vn, hn, _lib.current_stream()),
            "rv_generate_hypothesis_vanishing_point")
        return hypo

    @_lib.on_device(1)
    def voting_for_hypothesis(self, direct, coords, hypo_pts, inliers, inlier_thresh):
        tn, vn = self._dims(direct, coords)
        _check_cuda_contig(hypo_pts, "hypo_pts")
        _check_cuda_contig(inliers, "inliers")
        hn = hypo_pts.shape[0]
        assert tuple(hypo_pts.shape) == (hn, vn, 2) and tuple(inliers.shape) == (hn, vn, tn)
        assert inliers.dtype == torch.uint8
        _lib.check(_lib.lib().rv_voting_for_hypothesis(_lib.ptr(direct), _lib.ptr(coords), _lib.ptr(hypo_pts),
                                                       _lib.ptr(inliers), tn, vn, hn, float(inlier_thresh),
                                                       _lib.current_stream()), "rv_voting_for_hypothesis")

    @_lib.on_device(1)
    def voting_for_hypothesis_vanishing_point(self, direct, coords, hypo_pts, inliers, inlier_thresh):
        tn, vn = self._dims(direct, coords)
        _check_cuda_contig(hypo_pts, "hypo_pts")
        _check_cuda_contig(inliers, "inliers")
        hn = hypo_pts.shape[0]
        assert tuple(hypo_pts.shape) == (hn, vn, 3) and tuple(inliers.shape) == (hn, vn, tn)
        _lib.check(_lib.lib().rv_voting_for_hypothesis_vanishing_point(
            _lib.ptr(direct), _lib.ptr(coords), _lib.ptr(hypo_pts), _lib.ptr(inliers), tn, vn, hn, float(inlier_thresh),
            _lib.current_stream()), "rv_voting_for_hypothesis_vanishing_point")

    @_lib.on_device(1)
    def vote_count(self, direct, coords, hypo_pts, inlier_thresh, vanishing_point=False):
        """Fused vote + count (no [hn,vn,tn] mask): -> counts [hn,vn] int32."""
        tn, vn = self._dims(direct, coords)
        _check_cuda_contig(hypo_pts, "hypo_pts")
        hn = hypo_pts.shape[0]
        counts = torch.empty((hn, vn), dtype=torch.int32, device=direct.device)
        _lib.check(_lib.lib().rv_vote_count(_lib.ptr(direct), _lib.ptr(coords), _lib.ptr(hypo_pts), _lib.ptr(counts),
                                            tn, vn, hn, float(inlier_thresh), int(vanishing_point),
                                            _lib.current_stream()), "rv_vote_count")
        return counts


ransac_voting = _RansacVotingModule()


def _ransac_layer_call(mask, vertex, hn, inlier_thresh, min_num, max_num, idxs, seed, want_hyp=False, want_inliers=False):
    """One call of rv_ransac_voting_layer for the whole batch: compaction of the foreground, hypotheses, fused
    vote + count, per-keypoint winner, inlier set of the winner and its least-squares refit -- all on the device."""
    if not vertex.is_cuda:
        raise RuntimeError("ransac_voting_layer: CUDA tensors required (no CPU fallback)")
    dev = vertex.device
    b, h, w, vn, _ = vertex.shape
    m = mask.detach().to(device=dev).reshape(b, h, w)
    m = (m != 0).to(torch.float32).contiguous()
    vtx = vertex.detach().to(dtype=torch.float32).contiguous()
    L = _lib.lib()
    ws = torch.empty(L.rv_layer_workspace_bytes(b, h, w, vn, hn), dtype=torch.uint8, device=dev)
    win = torch.empty((b, vn, 2), dtype=torch.float32, device=dev)
    hyp = torch.empty((b, hn, vn, 2), dtype=torch.float32, device=dev) if want_hyp else None
    cnt = torch.empty((b, hn, vn), dtype=torch.int32, device=dev) if want_hyp else None
    tn = torch.empty((b,), dtype=torch.int32, device=dev) if (want_hyp or want_inliers) else None
    inl = torch.zeros((b, vn, h * w), dtype=torch.uint8, device=dev) if want_inliers else None
    ix = None
    if idxs is not None:
        ix = idxs.detach().to(device=dev, dtype=torch.int32).contiguous()
        assert tuple(ix.shape) == (b, hn, vn, 2), ix.shape
    if seed is None:
        seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())     # host RNG (torch.manual_seed reproducible), no device sync
    _lib.check(L.rv_ransac_voting_layer(_lib.ptr(m), _lib.ptr(vtx), b, h, w, vn, hn, float(inlier_thresh), int(min_num), int(max_num),
                                        int(seed) & 0xFFFFFFFF, _lib.ptr(ix), _lib.ptr(win), _lib.ptr(hyp), _lib.ptr(cnt), _lib.ptr(tn),
                                        _lib.ptr(inl), _lib.ptr(ws), ws.numel(), _lib.current_stream()), "rv_ransac_voting_layer")
    return win, hyp, cnt, tn, inl


@_lib.on_device(1)
def ransac_voting_layer(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20, min_num=5,
                        max_num=30000, idxs=None, seed=None, return_inliers=False):
    """ransac_voting_gpu.py:7-104 on the device: mask [b,h,w], vertex [b,h,w,vn,2] -> keypoints [b,vn,2].

    The reference draws its hypothesis pixel pairs ONCE per image, outside its `while` loop (:48), so every round
    regenerates the same hypotheses and counts and its strict `<` update never fires after round 1: `confidence` and
    `max_iter` only decide when that loop stops, not what it returns.  One device-side round is therefore the same
    function -- without the per-round device->host syncs, the [hn,vn,tn] inlier mask, torch.nonzero or torch.solve.
    ``idxs`` [b,hn,vn,2] int32 (optional, taken modulo the foreground count) replaces the on-device RNG (tests);
    ``return_inliers`` also returns (inlier mask [b,vn,h*w] u8 in compacted-pixel order, tn [b])."""
    del confidence, max_iter   # see the docstring: they do not influence the reference's result
    win, _, _, tn, inl = _ransac_layer_call(mask, vertex, int(round_hyp_num), inlier_thresh, min_num, max_num, idxs, seed,
                                            want_inliers=return_inliers)
    return (win, inl, tn) if return_inliers else win


def ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20, min_num=5,
                           max_num=30000, **kw):
    """ransac_voting_gpu.py:123-218: the v3 variant differs from ransac_voting_layer only in using bool masks and a
    batched inverse for the final 2x2 solves -- numerically the same function; same device-side implementation."""
    return ransac_voting_layer(mask, vertex, round_hyp_num, inlier_thresh, confidence, max_iter, min_num, max_num, **kw)


@_lib.on_device(1)
def b_inv(b_mat):
    """ransac_voting_gpu.py:107-120: batched matrix inverse used by the voting-distribution code; a singular batch falls back
    to the identity like the reference (its torch.solve call predates torch.linalg)."""
    eye = b_mat.new_ones(b_mat.size(-1)).diag().expand_as(b_mat)
    try:
        return torch.linalg.solve(b_mat, eye)
    except RuntimeError:   # singular input (https://github.com/zju3dv/clean-pvnet/issues/8)
        return eye


def estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=256, min_hyp_num=4096, topk=128,
                                           inlier_thresh=0.99, min_num=5, max_num=30000, output_hyp=False, seed=None):
    """ransac_voting_gpu.py:221-330: hypothesis cloud of `min_hyp_num` line intersections per keypoint, weighted by their
    inlier ratio (ratios more than 0.1 below the best are dropped) -> covariance around `mean` [b,vn,2].  The reference
    draws fresh pixel pairs for each of its ceil(min_hyp_num / round_hyp_num) rounds and concatenates them: here all
    hypotheses are generated and counted in one device call (mask == 1 is the foreground, :233)."""
    del topk, output_hyp
    b, h, w, vn, _ = vertex.shape
    hn = int(np.ceil(min_hyp_num / round_hyp_num)) * int(round_hyp_num)
    fg = (mask.reshape(b, h, w) == 1)
    _, hyp, cnt, tn, _ = _ransac_layer_call(fg, vertex, hn, inlier_thresh, min_num, max_num, None, seed, want_hyp=True)
    tnf = tn.to(torch.float32).clamp_min(1.0).view(b, 1, 1)
    ratio = cnt.to(torch.float32) / tnf                                       # [b,hn,vn]
    empty = (tn <= 0).view(b, 1, 1)
    ratio = torch.where(empty, torch.ones_like(ratio), ratio)                 # too few pixels: zeros / ones like the reference (:237-247)
    all_hyp = hyp.permute(0, 2, 1, 3)                                         # b,vn,hn,2
    all_ratio = ratio.permute(0, 2, 1).clone()                                # b,vn,hn
    thresh = torch.max(all_ratio, 2)[0] - 0.1
    all_ratio = torch.where(all_ratio < thresh.unsqueeze(2), torch.zeros_like(all_ratio), all_ratio)
    diff = all_hyp - mean.unsqueeze(2)
    cov = torch.matmul(diff.transpose(2, 3), diff * all_ratio.unsqueeze(3))
    cov = cov / (torch.sum(all_ratio, 2).unsqueeze(2).unsqueeze(3) + 1e-3)
    return mean, cov


# ------------------------------------------------------------------------------------------------ nnd
class _NndModule:
    """Drop-in for torch_nndistance_aten (nnd_cuda.cpp:86-89)."""

    @staticmethod
    @_lib.on_device(0)
    def nnd_forward_cuda(xyz1, xyz2, dist1, dist2, idx1, idx2):
        for t, n in ((xyz1, "xyz1"), (xyz2, "xyz2"), (dist1, "dist1"), (dist2, "dist2"), (idx1, "idx1"), (idx2, "idx2")):
            _check_cuda_contig(t, n)
        b, n, _ = xyz1.shape
        m = xyz2.shape[1]
        return _lib.lib().nnd_forward_cuda(_lib.ptr(xyz1), _lib.ptr(xyz2), _lib.ptr(dist1), _lib.ptr(dist2),
                                           _lib.ptr(idx1), _lib.ptr(idx2), b, n, m, _lib.current_stream())

    @staticmethod
    @_lib.on_device(0)
    def nnd_backward_cuda(xyz1, xyz2, gradxyz1, gradxyz2, graddist1, graddist2, idx1, idx2):
        b, n, _ = xyz1.shape
        m = xyz2.shape[1]
        return _lib.lib().nnd_backward_cuda(_lib.ptr(xyz1), _lib.ptr(xyz2), _lib.ptr(gradxyz1), _lib.ptr(gradxyz2),
                                            _lib.ptr(graddist1), _lib.ptr(graddist2), _lib.ptr(idx1), _lib.ptr(idx2),
                                            b, n, m, _lib.current_stream())


torch_nndistance_aten = _NndModule()


class NNDFunction(Function):
    """torch_nndistance.py:13-84."""

    @staticmethod
    def forward(ctx, xyz1, xyz2):
        if not xyz1.is_cuda:
            raise RuntimeError("nnd: CUDA tensors required (no CPU fallback)")
        xyz1 = xyz1.contiguous().float()
        xyz2 = xyz2.contiguous().float()
        b, n, _ = xyz1.size()
        m = xyz2.size(1)
        dist1 = torch.zeros(b, n, device=xyz1.device)
        dist2 = torch.zeros(b, m, device=xyz1.device)
        idx1 = torch.zeros(b, n, dtype=torch.int32, device=xyz1.device)
        idx2 = torch.zeros(b, m, dtype=torch.int32, device=xyz1.device)
        if torch_nndistance_aten.nnd_forward_cuda(xyz1, xyz2, dist1, dist2, idx1, idx2) != 1:
            raise _lib.GdrnError("nnd_forward_cuda failed: " + _lib.last_error())
        ctx.save_for_backward(xyz1, xyz2, dist1, dist2, idx1, idx2)
        return dist1, dist2

    @staticmethod
    def backward(ctx, graddist1, graddist2):
        xyz1, xyz2, dist1, dist2, idx1, idx2 = ctx.saved_tensors
        graddist1 = graddist1.contiguous()
        graddist2 = graddist2.contiguous()
        gradxyz1 = torch.zeros_like(xyz1)
        gradxyz2 = torch.zeros_like(xyz2)
        if torch_nndistance_aten.nnd_backward_cuda(xyz1, xyz2, gradxyz1, gradxyz2, graddist1, graddist2, idx1, idx2) != 1:
            raise _lib.GdrnError("nnd_backward_cuda failed: " + _lib.last_error())
        return gradxyz1, gradxyz2


def nnd(xyz1, xyz2):
    return NNDFunction.apply(xyz1, xyz2)


# ----------------------------------------------------------------------------------------------- flow
class _FlowModule:
    """Drop-in for flow_cuda (flow_cuda.cpp:30-47)."""

    @staticmethod
    @_lib.on_device(0)
    def forward(depth_src, depth_tgt, KT, Kinv):
        for t, n in ((depth_src, "depth_src"), (depth_tgt, "depth_tgt"), (KT, "KT"), (Kinv, "Kinv")):
            _check_cuda_contig(t, n)
        if depth_src.dtype != torch.float32:
            raise RuntimeError("flow_cuda.forward: float32 only on the CUDA path")
        B, _, H, W = depth_src.shape
        flow = torch.empty((B, 2, H, W), dtype=torch.float32, device=depth_src.device)
        valid = torch.empty((B, 1, H, W), dtype=torch.float32, device=depth_src.device)
        _lib.check(_lib.lib().flow_forward_cuda(_lib.ptr(depth_src), _lib.ptr(depth_tgt), _lib.ptr(KT), _lib.ptr(Kinv),
                                                _lib.ptr(flow), _lib.ptr(valid), B, H, W, _lib.current_stream()),
                   "flow_forward_cuda")
        return [flow, valid]


flow_cuda = _FlowModule()


def calc_se3_torch_batch(pose_src, pose_tgt):
    """core/utils/pose_utils.py calc_se3_torch_batch: T = pose_tgt * inv(pose_src), [B,3,4]."""
    R_s, t_s = pose_src[:, :3, :3], pose_src[:, :3, 3:4]
    R_t, t_t = pose_tgt[:, :3, :3], pose_tgt[:, :3, 3:4]
    R = R_t @ R_s.transpose(1, 2)
    t = t_t - R @ t_s
    return torch.cat([R, t], dim=2)


class FlowFunction(Function):
    """flow_torch.py:15-40."""

    @staticmethod
    def forward(ctx, depth_src, depth_tgt, pose_src, pose_tgt, K):
        se3 = calc_se3_torch_batch(pose_src, pose_tgt)
        KT = (K @ se3).contiguous()
        Kinv = K.inverse().contiguous()
        out = flow_cuda.forward(depth_src.contiguous(), depth_tgt.contiguous(), KT, Kinv)
        return out[0], out[1]


flow = FlowFunction.apply


# ------------------------------------------------------------------------------------ uncertainty pnp
def uncertainty_pnp_refine(points_2d, weights_2d, points_3d, camera_matrix, init_rt):
    """The compiled part of un_pnp_utils.uncertainty_pnp (lib.uncertainty_pnp): host f64 arrays -> result_rt [6]."""
    pn = points_2d.shape[0]
    a2 = np.ascontiguousarray(points_2d, np.float64)
    a3 = np.ascontiguousarray(points_3d, np.float64)
    aw = np.ascontiguousarray(weights_2d, np.float64)
    aK = np.ascontiguousarray(camera_matrix, np.float64)
    ai = np.ascontiguousarray(init_rt, np.float64).reshape(6)
    res = np.empty([6], np.float64)
    c = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    _lib.lib().uncertainty_pnp(c(a2), c(a3), c(aw), c(aK), c(ai), c(res), pn)
    return res


def uncertainty_pnp(points_2d, weights_2d, points_3d, camera_matrix):
    """un_pnp_utils.py:11-78: EPnP on the 4 highest-weight points (cv2, host) then weighted LM refine -> [3,4]."""
    import cv2

    pn = points_2d.shape[0]
    assert points_3d.shape[0] == pn and pn >= 4
    dist_coeffs = np.zeros(shape=[8, 1], dtype=np.float64)
    points_3d = points_3d.astype(np.float64)
    points_2d = points_2d.astype(np.float64)
    weights_2d = weights_2d.astype(np.float64)
    camera_matrix = camera_matrix.astype(np.float64)
    idxs = np.argsort(weights_2d[:, 0] + weights_2d[:, 1])[-4:]
    _, R_exp, t = cv2.solvePnP(np.expand_dims(points_3d[idxs, :], 0), np.expand_dims(points_2d[idxs, :], 0),
                               camera_matrix, dist_coeffs, None, None, False, flags=cv2.SOLVEPNP_EPNP)
    if pn == 4:
        R, _ = cv2.Rodrigues(R_exp)
        return np.concatenate([R, t], axis=-1)
    init_rt = np.concatenate([R_exp, t], 0)
    result_rt = uncertainty_pnp_refine(points_2d, weights_2d, points_3d, camera_matrix, init_rt)
    R, _ = cv2.Rodrigues(result_rt[:3])
    return np.concatenate([R, result_rt[3:, None]], axis=-1)


def covariance_weights(covars):
    """Per-point scalar weights of uncertainty_pnp_v2 (un_pnp_utils.py:96-104): 1 / (largest eigenvalue of the 2x2 covariance),
    0 where the covariance is degenerate (covars[i, 0, 0] < 1e-5).  covars [pn,2,2] -> float64 [pn]."""
    covars = np.asarray(covars)
    lam = np.linalg.eigvals(covars.astype(np.float64)).real.max(axis=-1)        # [pn] largest eigenvalue of each covariance
    ok = covars[:, 0, 0] >= 1e-5
    return np.where(ok, 1.0 / np.where(ok, lam, 1.0), 0.0)


def uncertainty_pnp_v2(points_2d, covars, points_3d, camera_matrix, type="single"):
    """un_pnp_utils.py:81-158: the covariance form.  Every 2-D point carries a 2x2 covariance; its weight is the inverse of the
    LARGEST eigenvalue (0 for a degenerate covariance, covars[i,0,0] < 1e-5), used isotropically ([w, 0, w] rows); EPnP on the
    four highest-weight points, then the same weighted LM refine as uncertainty_pnp -> [3,4].  `type` is accepted and unused,
    as in the reference."""
    import cv2

    pn = points_2d.shape[0]
    assert points_3d.shape[0] == pn and pn >= 4 and covars.shape[0] == pn
    points_3d = points_3d.astype(np.float64)
    points_2d = points_2d.astype(np.float64)
    camera_matrix = camera_matrix.astype(np.float64)
    w = covariance_weights(covars)
    idxs = np.argsort(w)[-4:]
    dist_coeffs = np.zeros(shape=[8, 1], dtype=np.float64)
    _, R_exp, t = cv2.solvePnP(np.expand_dims(points_3d[idxs, :], 0), np.expand_dims(points_2d[idxs, :], 0),
                               camera_matrix, dist_coeffs, None, None, False, flags=cv2.SOLVEPNP_EPNP)
    if pn == 4:
        R, _ = cv2.Rodrigues(R_exp)
        return np.concatenate([R, t], axis=-1)
    weights_2d = np.stack([w, np.zeros(pn), w], axis=1)
    result_rt = uncertainty_pnp_refine(points_2d, weights_2d, points_3d, camera_matrix, np.concatenate([R_exp, t], 0))
    R, _ = cv2.Rodrigues(result_rt[:3])
    return np.concatenate([R, result_rt[3:, None]], axis=-1)


@_lib.on_device(0)
def uncertainty_pnp_batched(pts2d, pts3d, wgt2d, K, init_rt):
    """Device batched refine: pts2d [n,pn,2], pts3d [n,pn,3], wgt2d [n,pn,3], K [n,3,3], init_rt [n,6] (f64 CUDA)."""
    n, pn, _ = pts2d.shape
    ts = [t.to(torch.float64).contiguous() for t in (pts2d, pts3d, wgt2d, K, init_rt)]
    res = torch.empty((n, 6), dtype=torch.float64, device=pts2d.device)
    _lib.check(_lib.lib().upnp_batched(*[_lib.ptr(t) for t in ts], _lib.ptr(res), pn, n, _lib.current_stream()),
               "upnp_batched")
    return res


# ---------------------------------------------------------------------------------------------------------------
# ROI crop + resize (core/utils/data_utils.py:115-189: crop_resize_by_warp_affine, get_affine_transform)
# ---------------------------------------------------------------------------------------------------------------
def get_affine_transform(center, scale, rot, output_size, shift=(0.0, 0.0), inv=False):
    """2x3 float64 forward matrix, same contract as the reference's get_affine_transform (data_utils.py:136-189):
    the affine map taking (center, center + rotated (0, -scale_w/2), their perpendicular third point) onto
    (out centre, out centre + (0, -out_w/2), third point).  The reference builds the three point pairs in float32
    and solves with cv2.getAffineTransform; here the same float32 point pairs are solved in closed form in float64
    (equal to 1e-12; the warp quantises coordinates to 1/32 pixel, so crops are identical)."""
    # dtype handling as in the reference: tuples / lists and python scalars become float32, arrays keep their dtype, so that
    # `center + src_dir + scale * shift` is evaluated at the caller's precision and rounded ONCE into the float32 points
    center = np.array(center, np.float32) if isinstance(center, (tuple, list)) else np.asarray(center)
    if np.isscalar(scale):
        scale = np.array([scale, scale], np.float32)
    scale = np.asarray(scale)
    if np.isscalar(output_size):
        output_size = (output_size, output_size)
    shift = np.array(shift, np.float32) if isinstance(shift, (tuple, list)) else np.asarray(shift)
    src_w, dst_w, dst_h = scale[0], output_size[0], output_size[1]
    rot_rad = np.pi * rot / 180
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)
    src_dir = np.array([0 * cs - (src_w * -0.5) * sn, 0 * sn + (src_w * -0.5) * cs])
    dst_dir = np.array([0, dst_w * -0.5], np.float32)
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0, :] = center + scale * shift
    src[1, :] = center + src_dir + scale * shift
    dst[0, :] = [dst_w * 0.5, dst_h * 0.5]
    dst[1, :] = np.array([dst_w * 0.5, dst_h * 0.5], np.float32) + dst_dir

    def third(a, b):
        d = a - b
        return b + np.array([-d[1], d[0]], np.float32)

    src[2, :] = third(src[0], src[1])
    dst[2, :] = third(dst[0], dst[1])
    a, b = (dst, src) if inv else (src, dst)
    A = np.concatenate([a.astype(np.float64), np.ones((3, 1))], axis=1)   # [3,3]: rows (x, y, 1)
    return np.linalg.solve(A, b.astype(np.float64)).T.copy()               # [2,3]


def _affine_batch(M, device):
    if torch.is_tensor(M):   # already on the device (a caller that batches its uploads): [n,2,3] / [n,6] float64
        Md = M.detach().to(device=device, dtype=torch.float64).reshape(-1, 6).contiguous()
        return Md, Md.shape[0]
    M = np.ascontiguousarray(np.asarray(M, np.float64).reshape(-1, 6))
    return torch.from_numpy(M).to(device), M.shape[0]


@_lib.on_device(0)
def crop_resize_image(image, M, output_size, pixel_mean=(0.0, 0.0, 0.0), pixel_std=(255.0, 255.0, 255.0), out=None):
    """Batched cv2.warpAffine(image, M[i], (w, h), INTER_LINEAR) + normalize_image for an HxWxC uint8 CUDA image:
    returns roi_img [n, C, h, w] float32 (predictor_gdrn.py:417-422).  M: [n,2,3] float64 forward transforms (numpy, or
    a CUDA tensor).  out: optional preallocated [n,C,h,w] float32 CUDA tensor (static CUDA-graph input buffers)."""
    _check_cuda_contig(image, "image")
    assert image.dtype == torch.uint8 and image.dim() == 3
    H, W, C = image.shape
    ow, oh = (output_size, output_size) if np.isscalar(output_size) else output_size
    Md, n = _affine_batch(M, image.device)
    if out is None:
        out = torch.empty((n, C, int(oh), int(ow)), dtype=torch.float32, device=image.device)
    else:
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (n, C, int(oh), int(ow))
    mean = (ctypes.c_double * C)(*[float(v) for v in list(pixel_mean)[:C]])
    std = (ctypes.c_double * C)(*[float(v) for v in list(pixel_std)[:C]])
    _lib.check(_lib.lib().gdrn_crop_resize_u8(_lib.ptr(image), H, W, C, _lib.ptr(Md), n, int(oh), int(ow), mean, std,
                                              _lib.ptr(out), _lib.current_stream()), "gdrn_crop_resize_u8")
    return out


@_lib.on_device(0)
def crop_resize_float(src, M, output_size, nearest=False, out=None):
    """Batched cv2.warpAffine on an HxW(xC) float32 CUDA array (INTER_LINEAR, or INTER_NEAREST for depth):
    returns [n, C, h, w] float32 (roi_coord_2d / roi_depth, predictor_gdrn.py:425-438).  M / out as in crop_resize_image."""
    _check_cuda_contig(src, "src")
    assert src.dtype == torch.float32 and src.dim() in (2, 3)
    H, W = src.shape[:2]
    C = 1 if src.dim() == 2 else src.shape[2]
    ow, oh = (output_size, output_size) if np.isscalar(output_size) else output_size
    Md, n = _affine_batch(M, src.device)
    if out is None:
        out = torch.empty((n, C, int(oh), int(ow)), dtype=torch.float32, device=src.device)
    else:
        assert out.is_cuda and out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (n, C, int(oh), int(ow))
    _lib.check(_lib.lib().gdrn_crop_resize_f32(_lib.ptr(src), H, W, C, _lib.ptr(Md), n, int(oh), int(ow), int(bool(nearest)),
                                               _lib.ptr(out), _lib.current_stream()), "gdrn_crop_resize_f32")
    return out


# ---------------------------------------------------------------------------------------------------------------
# Model inputs for the ROIs of many images (read_data_test + batch_data_test, datasets/data_loader.py:751-797,
# engine/engine_utils.py:213-241) in two launches: csrc/roi_batch.cu
# ---------------------------------------------------------------------------------------------------------------
ROI_BATCH_KEYS = (("roi_center", (2,), torch.float32), ("roi_wh", (2,), torch.float32), ("scale", (), torch.float32),
                  ("resize_ratio", (), torch.float32), ("roi_extent", (3,), torch.float32), ("roi_cam", (3, 3), torch.float32),
                  ("roi_cls", (), torch.int64), ("im_H", (), torch.float32), ("im_W", (), torch.float32),
                  ("bbox_est", (4,), torch.float32), ("M_in", (6,), torch.float64), ("M_out", (6,), torch.float64))


def roi_batch_buffers(n, device, input_res=256, output_res=64, with_depth=False):
    """Preallocated outputs of roi_batch_inputs for n ROIs (static buffers a CUDA graph can be captured over)."""
    z = lambda shape, dtype=torch.float32: torch.zeros((n,) + tuple(shape), dtype=dtype, device=device)
    out = {k: z(shape, dtype) for k, shape, dtype in ROI_BATCH_KEYS}
    out["roi_img"] = z((3, input_res, input_res))
    out["roi_coord_2d"] = z((2, output_res, output_res))
    if with_depth:
        out["roi_depth"] = z((1, input_res, input_res))
        out["depth_sensor"] = z((output_res, output_res))
    return out


@_lib.on_device(0)
def roi_batch_inputs(images, dets, Ks, extents, dzi_pad_scale=1.5, input_res=256, output_res=64,
                     pixel_mean=(0.0, 0.0, 0.0), pixel_std=(255.0, 255.0, 255.0), depth=None, depth_factor=None, out=None):
    """The model inputs of a batch of images, as batch_data_test returns them, from two kernels (gdrn_roi_setup +
    gdrn_roi_crop_multi) on the current stream; no allocation when ``out`` is given, no synchronisation.

    images [N,H,W,C] uint8 CUDA (BGR, C = 1 or 3; one call per image size); dets: mapping with "det_meta" [n,2] int32
    (image index, label) and "bbox_est" [n,4] float32 XYWH_ABS (CUDA), plus optional "score" / "time" [n] passed
    through; Ks [N,3,3] float32 CUDA; extents [nc,3] float32 CUDA (per label); depth [N,H,W] uint16 CUDA with
    depth_factor [N] float64 CUDA (1000 / depth_scale) adds roi_depth [n,1,in,in] and the 64x64 depth-refine sensor crop
    ("depth_sensor" [n,out,out]).  Returns a dict: roi_img, roi_coord_2d, roi_center, roi_wh, scale, resize_ratio,
    roi_extent, roi_cam, roi_cls (int64), im_H, im_W, bbox_est (XYXY), M_in / M_out [n,6] float64 and the pass-through
    keys.  Image indices and labels are validated by the caller (they come from host data)."""
    _check_cuda_contig(images, "images")
    if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] not in (1, 3):
        raise ValueError(f"images must be [N,H,W,1|3] uint8, got {tuple(images.shape)} {images.dtype}")
    N, H, W, C = images.shape
    meta, xywh = dets["det_meta"], dets["bbox_est"]
    for t, name, dt in ((meta, "det_meta", torch.int32), (xywh, "bbox_est", torch.float32), (Ks, "Ks", torch.float32),
                        (extents, "extents", torch.float32)):
        _check_cuda_contig(t, name)
        if t.dtype != dt:
            raise ValueError(f"{name} must be {dt}")
    n = meta.shape[0]
    if tuple(Ks.shape) != (N, 3, 3):
        raise ValueError(f"Ks must be [{N},3,3], got {tuple(Ks.shape)}")
    with_depth = depth is not None
    if with_depth:
        _check_cuda_contig(depth, "depth")
        _check_cuda_contig(depth_factor, "depth_factor")
        if depth.dtype != torch.uint16 or tuple(depth.shape) != (N, H, W) or depth_factor.dtype != torch.float64:
            raise ValueError("depth must be [N,H,W] uint16 with depth_factor [N] float64")
    if out is None:
        out = roi_batch_buffers(n, images.device, input_res, output_res, with_depth)
    im_hw = torch.full((max(N, 1), 2), H, dtype=torch.int32, device=images.device)   # device fills: no host copy
    im_hw[:, 1].fill_(W)
    p = _lib.ptr
    L = _lib.lib()
    _lib.check(L.gdrn_roi_setup(p(meta), p(xywh), n, p(Ks), p(im_hw), p(extents), float(dzi_pad_scale), int(input_res),
                                int(output_res), *[p(out[k]) for k, _, _ in ROI_BATCH_KEYS], _lib.current_stream()),
               "gdrn_roi_setup")
    mean = (ctypes.c_double * 3)(*[float(v) for v in pixel_mean])
    std = (ctypes.c_double * 3)(*[float(v) for v in pixel_std])
    _lib.check(L.gdrn_roi_crop_multi(p(images), H, W, C, p(meta), p(out["M_in"]), p(out["M_out"]), n, int(input_res),
                                     int(output_res), mean, std, p(depth) if with_depth else None,
                                     p(depth_factor) if with_depth else None, p(out["roi_img"]), p(out["roi_coord_2d"]),
                                     p(out.get("roi_depth")) if with_depth else None,
                                     p(out.get("depth_sensor")) if with_depth else None, _lib.current_stream()),
               "gdrn_roi_crop_multi")
    res = dict(out)
    for k in ("score", "time"):
        if k in dets:
            res[k] = dets[k]
    return res
