"""Network-initialised PnP (TEST.PNP_TYPE = net_iter_pnp / net_ransac_pnp / net_ransac_pnp_rot) and coor-z depth refine
(TEST.USE_COOR_Z_REFINE) against the reference's recipes restated on the host: cv2.solvePnP / solvePnPRansac called the
way process_net_and_pnp calls them (engine/gdrn_evaluator.py:241-371), and numpy for gdrn_evaluator.py:528-561."""
import numpy as np
import pytest
import torch

from oracle import gdrn_model_oracle as O
from oracle import ops_oracle as OO
from oracle import pnp_oracle as PO

K_CAM = np.array([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]])
NET_TYPES = ("net_iter_pnp", "net_ransac_pnp", "net_ransac_pnp_rot")


def _rot(axis, angle):
    return O.axangle2mat(np.asarray(axis, np.float64) / np.linalg.norm(axis), angle)


def _rot_err(Ra, Rb):
    """Angle of Ra^T Rb in radians, accurate near 0 (sin from the skew part)."""
    D = Ra.T @ Rb
    s = 0.5 * np.linalg.norm([D[2, 1] - D[1, 2], D[0, 2] - D[2, 0], D[1, 0] - D[0, 1]])
    return float(np.arctan2(s, 0.5 * (np.trace(D) - 1)))


# ------------------------------------------------------------------------------------------------ host oracles
def ref_net_pnp(points_3d, points_2d, K, rot_est_net, out_transes, i, pnp_type):
    """gdrn_evaluator.py:316-358 for ROI i: `out_transes` is the float32 [n,3] array the reference reads the network
    translations into, and trans_est_net is its row VIEW -- cv2.solvePnP writes its result into it in place.
    Returns (R, t, retval of the cv2 call or None when < 4 points)."""
    import cv2

    trans_est_net = out_transes[i]
    if len(points_2d) < 4:
        return rot_est_net, trans_est_net.copy(), None
    dist_coeffs = np.zeros(shape=[8, 1], dtype="float64")
    points_2d = np.ascontiguousarray(points_2d.astype(np.float64))
    points_3d = np.ascontiguousarray(points_3d.astype(np.float64))
    camera_matrix = K.astype(np.float64)
    rvec0, _ = cv2.Rodrigues(rot_est_net)
    if pnp_type in ("net_ransac_pnp", "net_ransac_pnp_rot"):
        ok, rvec, t_est, _ = cv2.solvePnPRansac(objectPoints=points_3d[None], imagePoints=points_2d[None], cameraMatrix=camera_matrix,
                                                distCoeffs=dist_coeffs, flags=cv2.SOLVEPNP_EPNP, useExtrinsicGuess=True, rvec=rvec0,
                                                tvec=trans_est_net, reprojectionError=3.0, iterationsCount=20)
    else:
        ok, rvec, t_est = cv2.solvePnP(objectPoints=points_3d, imagePoints=points_2d, cameraMatrix=camera_matrix, distCoeffs=dist_coeffs,
                                       flags=cv2.SOLVEPNP_ITERATIVE, useExtrinsicGuess=True, rvec=rvec0, tvec=trans_est_net)
    rot_est, _ = cv2.Rodrigues(rvec)
    if pnp_type != "net_ransac_pnp_rot":
        if np.linalg.norm(np.asarray(t_est, np.float64).reshape(3) - np.asarray(trans_est_net, np.float64).reshape(3)) > 1:
            t_est = trans_est_net
    else:
        t_est = trans_est_net
    return rot_est, np.asarray(t_est, np.float64).reshape(3), ok


def ref_correspondences(cx, cy, cz, m, c2d, ext, imH, imW, mask_thr=0.5):
    """get_out_mask (L1) + get_img_model_points_with_coords2d (gdrn_evaluator.py:1183-1221) on float32 maps."""
    return PO.correspondences(cx, cy, cz, m, c2d, ext, imH, imW, mask_thr)[:2]


def ref_coor_z_step(xyz01, mask_n, sensor, ren, K_crop, rot_est, trans, thresh=0.8):
    """One fast-depth-refine iteration with TEST.USE_COOR_Z_REFINE (gdrn_evaluator.py:528-561): xyz01 [h,w,3] raw
    coordinate maps, mask_n [h,w] normalised mask, rot_est float32 [3,3]."""
    crop_res = mask_n.shape[0]
    coor_np_r = (rot_est @ xyz01.reshape(-1, 3).T).T.reshape(crop_res, crop_res, 3)
    query_img_norm = coor_np_r[:, :, -1] * mask_n
    query_img_norm = query_img_norm * (ren > 0) * (sensor > 0)
    norm_sum = query_img_norm.sum()
    if norm_sum == 0:
        return trans.copy()
    query_img_norm /= norm_sum
    norm_mask = query_img_norm > (query_img_norm.max() * thresh)
    yy, xx = np.argwhere(norm_mask).T
    depth_adjustment = np.median(sensor[yy, xx] - ren[yy, xx])
    yx_coords = np.stack(np.meshgrid(np.arange(crop_res), np.arange(crop_res))[::-1], axis=-1)
    yx_ray_2d = (yx_coords * query_img_norm[..., None]).sum(axis=(0, 1))
    ray_3d = np.linalg.inv(K_crop) @ (*yx_ray_2d[::-1], 1)
    ray_3d /= ray_3d[2]
    return trans + (ray_3d[:, None] * depth_adjustment).reshape(3)


# ------------------------------------------------------------------------------------------------ synthetic inputs
def make_pnp_problem(rs, npts, outlier_frac, start):
    """Model points in a 12x20x9 cm box seen at 0.7-1.2 m, 0.5 px noise, `outlier_frac` gross outliers; initial pose
    perturbed by 2-10 deg and a few cm ("perturbed") or the identity rotation at the true t ("identity")."""
    if start == "identity":
        R = _rot(rs.randn(3), 0.3 + 0.5 * rs.rand())
    else:
        R = _rot(rs.randn(3), rs.rand() * 3)
    t = np.array([rs.randn() * 0.05, rs.randn() * 0.05, 0.7 + rs.rand() * 0.5])
    X = (rs.rand(npts, 3) - 0.5) * np.array([0.12, 0.2, 0.09])
    xc = X @ R.T + t
    uv = np.stack([K_CAM[0, 0] * xc[:, 0] / xc[:, 2] + K_CAM[0, 2], K_CAM[1, 1] * xc[:, 1] / xc[:, 2] + K_CAM[1, 2]], 1)
    uv += rs.randn(npts, 2) * 0.5
    out = rs.rand(npts) < outlier_frac
    uv[out] += rs.randn(int(out.sum()), 2) * 40 + 25
    if start == "identity":
        R0, t0 = np.eye(3), t.copy()
    else:
        R0 = _rot(rs.randn(3), np.deg2rad(2 + 8 * rs.rand())) @ R
        t0 = t + rs.randn(3) * 0.03
    return X.astype(np.float32), uv.astype(np.float32), R0.astype(np.float32), t0.astype(np.float32)


def make_roi_maps(rs, hw=64, imH=480, imW=640):
    """Coordinate / mask maps of a sphere-shaped object seen through a ROI grid (the recipe of the RANSAC-PnP map test),
    with per-ROI network poses.  ROI roles: 0 plain; 1 network t at z = 2.0 m for an object at ~0.8 m; 2 empty mask;
    3 six pure-noise correspondences (no RANSAC model); 4 plain with a 6 deg network rotation error."""
    n = 5
    cx_, cy_, cz_, mk, c2d, ext, Rn, tn, GT = [], [], [], [], [], [], [], [], []
    for i in range(n):
        R = _rot(rs.randn(3), rs.rand() * 3)
        t = np.array([rs.randn() * 0.05, rs.randn() * 0.05, 0.75 + rs.rand() * 0.1])
        r_obj, e = 0.05, np.array([0.12, 0.13, 0.11])
        pc = K_CAM @ t
        pc = pc[:2] / pc[2]
        scale = 2.6 * r_obj * K_CAM[0, 0] / t[2]
        U, V = np.meshgrid(pc[0] + (np.arange(hw) - hw / 2) * scale / hw, pc[1] + (np.arange(hw) - hw / 2) * scale / hw)
        rays = np.stack([(U - K_CAM[0, 2]) / K_CAM[0, 0], (V - K_CAM[1, 2]) / K_CAM[1, 1], np.ones_like(U)], -1)
        rays /= np.linalg.norm(rays, axis=-1, keepdims=True)
        b_ = (rays * t).sum(-1)
        disc = b_ ** 2 - (t @ t - r_obj ** 2)
        hit = disc > 0
        Xc = rays * (b_ - np.sqrt(np.where(hit, disc, 0)))[..., None]
        coor = (Xc - t) @ R / e + 0.5 + rs.randn(hw, hw, 3) * 0.002
        coor[~hit] = 0.5
        m = np.where(hit, 0.9, 0.05) + rs.randn(hw, hw) * 0.02
        if i == 2:
            m[:] = 0.1; m[0, 0] = 0.2; coor[:] = 0.5
        if i == 3:
            m[:] = 0.05; coor[:] = 0.5
            for k, (r, c) in enumerate(((3, 5), (10, 50), (30, 20), (45, 60), (60, 8), (52, 33))):
                m[r, c] = 0.9
                coor[r, c] = rs.rand(3)
        t_net = t + rs.randn(3) * 0.01
        R_net = _rot(rs.randn(3), np.deg2rad(6 if i == 4 else 2)) @ R
        if i == 1:
            t_net = np.array([t[0], t[1], 2.0])
        cx_.append(coor[..., 0]); cy_.append(coor[..., 1]); cz_.append(coor[..., 2]); mk.append(m)
        c2d.append(np.stack([U / imW, V / imH])); ext.append(e); Rn.append(R_net); tn.append(t_net); GT.append((R, t))
    f32 = lambda a: np.stack(a).astype(np.float32)
    return dict(cx=f32(cx_), cy=f32(cy_), cz=f32(cz_), m=f32(mk), c2d=f32(c2d), ext=f32(ext), Rn=f32(Rn), tn=f32(tn), GT=GT,
                imH=imH, imW=imW)


# ------------------------------------------------------------------------------------------------ tests
def test_pnp_net_unknown_type_raises():
    from gdrnpp_bop2022_b200.pnp_ransac import pnp_net_from_maps

    with pytest.raises(NotImplementedError):
        pnp_net_from_maps(*([None] * 11), pnp_type="net_epnp")


@pytest.mark.gpu
@pytest.mark.parametrize("npts", [4, 5, 64, 600, 4096])
def test_solve_pnp_iterative_vs_cv2(dev, npts):
    """solve_pnp_iterative == cv2.solvePnP(ITERATIVE, useExtrinsicGuess=True) on the same float32 correspondences:
    both reach the same LM minimiser, R within 1e-5 rad and t within 1e-5 m.  0.5 px noise, 0-30 % gross outliers
    (>= 64 points), starts perturbed by 2-10 deg and a few cm plus one identity-rotation start."""
    import cv2

    from gdrnpp_bop2022_b200.pnp_ransac import solve_pnp_iterative

    rs = np.random.RandomState(100 + npts)
    starts = ["perturbed"] * 4 + ["identity"]
    probs = [make_pnp_problem(rs, npts, (0.0, 0.1, 0.2, 0.3, 0.15)[k] if npts >= 64 else 0.0, s) for k, s in enumerate(starts)]
    P3, P2, R0, t0 = (np.stack([p[j] for p in probs]) for j in range(4))
    T = lambda a: torch.from_numpy(a).to(dev)
    Ks = torch.from_numpy(K_CAM.astype(np.float32))[None].expand(len(probs), 3, 3)
    got = solve_pnp_iterative(T(P3), T(P2), Ks.to(dev), T(R0), T(t0)).cpu().numpy().astype(np.float64)
    for i in range(len(probs)):
        ok, rvec, tvec = cv2.solvePnP(P3[i].astype(np.float64), P2[i].astype(np.float64), K_CAM.astype(np.float32).astype(np.float64),
                                      np.zeros((8, 1)), rvec=cv2.Rodrigues(R0[i].astype(np.float64))[0],
                                      tvec=t0[i].astype(np.float64).reshape(3, 1), useExtrinsicGuess=True, flags=cv2.SOLVEPNP_ITERATIVE)
        assert ok
        Rc = cv2.Rodrigues(rvec)[0]
        assert _rot_err(got[i, :, :3], Rc) < 1e-5 and np.abs(got[i, :, 3] - tvec[:, 0]).max() < 1e-5, \
            (i, starts[i], _rot_err(got[i, :, :3], Rc), np.abs(got[i, :, 3] - tvec[:, 0]).max())
    # fewer than 4 points: the initial pose comes back unchanged
    few = solve_pnp_iterative(T(P3[:1, :3]), T(P2[:1, :3]), Ks[:1].to(dev), T(R0[:1]), T(t0[:1])).cpu()
    assert torch.equal(few[0, :, :3], torch.from_numpy(R0[0])) and torch.equal(few[0, :, 3], torch.from_numpy(t0[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("pnp_type", NET_TYPES)
def test_pnp_net_from_maps_vs_reference_recipe(dev, pnp_type):
    """pnp_net_from_maps vs process_net_and_pnp restated on the host on the same float32 maps (see make_roi_maps for
    the ROI roles): empty mask -> network pose bit-equal; no RANSAC model -> network pose; network t 1.2 m off -> the
    net t for net_ransac_pnp (the 1 m guard) but the PnP t for net_iter_pnp (the guard never fires there);
    net_ransac_pnp_rot -> t_net exactly."""
    from gdrnpp_bop2022_b200.pnp_ransac import pnp_net_from_maps

    d = make_roi_maps(np.random.RandomState(21))
    n = d["cx"].shape[0]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Ks = torch.from_numpy(K_CAM.astype(np.float32))[None].repeat(n, 1, 1).to(dev)
    poses, used = pnp_net_from_maps(T(d["cx"][:, None]), T(d["cy"][:, None]), T(d["cz"][:, None]), T(d["m"][:, None]), T(d["c2d"]),
                                    torch.full((n,), d["imH"]), torch.full((n,), d["imW"]), T(d["ext"]), Ks, T(d["Rn"]), T(d["tn"]),
                                    pnp_type=pnp_type, return_used=True)
    poses, used = poses.cpu().numpy(), used.cpu().numpy()
    out_transes = d["tn"].copy()            # the reference's float32 [n,3] array of network translations
    for i in range(n):
        p3, p2 = ref_correspondences(d["cx"][i], d["cy"][i], d["cz"][i], d["m"][i], d["c2d"][i], d["ext"][i], d["imH"], d["imW"])
        Rr, tr, ok = ref_net_pnp(p3, p2, K_CAM.astype(np.float32), d["Rn"][i], out_transes, i, pnp_type)
        R, t = poses[i, :, :3].astype(np.float64), poses[i, :, 3].astype(np.float64)
        if i == 2:        # empty mask: the network pose, bit-equal
            assert ok is None and np.array_equal(poses[i, :, :3], d["Rn"][i]) and np.array_equal(poses[i, :, 3], d["tn"][i])
            assert used[i] == 0
            continue
        if i == 3:
            assert len(p3) == 6
            if pnp_type == "net_iter_pnp":   # LM on six random correspondences: no reference behaviour to pin beyond this
                assert np.isfinite(poses[i]).all() and used[i] == 6
                continue
            # cv2 found no model (retval False) and does not write its outputs, so the reference's pose is undefined
            # here; the library returns the network pose, the guess the call was given
            assert ok is False
            assert np.array_equal(poses[i, :, :3], d["Rn"][i]) and np.array_equal(poses[i, :, 3], d["tn"][i]) and used[i] == 0
            continue
        assert ok and used[i] > 100
        if pnp_type == "net_iter_pnp":     # same LM minimiser as cv2's iterative solver
            assert _rot_err(R, Rr) < 1e-5 and np.abs(t - tr).max() < 1e-5, (i, _rot_err(R, Rr), np.abs(t - tr).max())
            if i == 1:                     # converged from z = 2.0 to the object; the reference keeps this t too
                assert abs(t[2] - d["GT"][i][1][2]) < 5e-3
        else:                              # RANSAC: same tolerance as the RANSAC-PnP map test
            assert _rot_err(R, Rr) < 0.02, (i, _rot_err(R, Rr))
            if pnp_type == "net_ransac_pnp_rot" or i == 1:
                assert np.array_equal(poses[i, :, 3], d["tn"][i]) and np.array_equal(tr, d["tn"][i].astype(np.float64))
            else:
                assert np.abs(t - tr).max() < 5e-3 and np.abs(t - d["tn"][i]).max() > 0


def _coor_z_inputs(seed, n=4, hw=64):
    rs = np.random.RandomState(seed)
    xyz = rs.rand(n, 3, hw, hw).astype(np.float32)
    mask = rs.rand(n, hw, hw).astype(np.float32)
    ren = np.where(rs.rand(n, hw, hw) < 0.7, 0.7 + 0.1 * rs.rand(n, hw, hw), 0).astype(np.float32)
    sensor = np.where(rs.rand(n, hw, hw) < 0.9, ren + 0.01 * rs.randn(n, hw, hw) + 0.02, 0).astype(np.float32)
    K = np.stack([np.array([[110.0 + 10 * rs.rand(), 0, 32 + rs.randn()], [0, 112.0, 31 + rs.randn()], [0, 0, 1]]) for _ in range(n)])
    h = np.float32(np.sqrt(0.5))
    rots = [_rot([0.0, 1.0, 0.0], 0.4),                               # (R xyz)_z = -0.39 x + 0.92 z: mixed signs, positive sum
            _rot([1.0, 0.0, 0.0], np.pi),                             # (R xyz)_z = -z: all weights <= 0, negative sum
            _rot([0.3, 1.0, 0.1], 2.2),                               # mixed signs, whatever the sum
            np.array([[-h, 0, -h], [0, 1, 0], [h, 0, -h]])]           # (R xyz)_z = h (x - z): cancels exactly below
    R = np.stack(rots).astype(np.float32)
    # ROI 3: two valid pixels with h*0.5 and -h*0.5 -> the weights sum to exactly 0
    mask[3] = 0; mask[3, 10, 10] = 1; mask[3, 40, 41] = 1
    xyz[3, :, 10, 10] = (0.5, 0.3, 0.0); xyz[3, :, 40, 41] = (0.0, 0.7, 0.5)
    for r, c in ((10, 10), (40, 41)):
        ren[3, r, c], sensor[3, r, c] = 0.75, 0.77
    t = np.stack([np.array([0.01, -0.02, 0.75]) + 0.01 * rs.randn(3) for _ in range(n)]).astype(np.float32)
    return xyz, mask, ren, sensor, K.astype(np.float32), R, t


@pytest.mark.gpu
def test_coor_z_single_refine_entry_vs_numpy(dev):
    """gdrn_depth_refine_step(weight_mode=1) == the reference's coor-z iteration restated in numpy, with negative
    weights, a negative sum (the cut then comes from the most negative weight) and an exactly-zero sum (pose unchanged);
    weight_mode 0 ignores the rotations."""
    from gdrnpp_bop2022_b200 import _lib as L

    xyz, mask, ren, sensor, K, R, t = _coor_z_inputs(3)
    n, hw = mask.shape[0], mask.shape[-1]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    xyz_d, mask_d, ren_d, sen_d, K_d, R_d = T(xyz), T(mask), T(ren), T(sensor), T(K), T(R)
    stream = L.current_stream()

    def run(rot, mode):
        out = T(t).clone()
        L.check(L.lib().gdrn_depth_refine_step(L.ptr(xyz_d), L.ptr(mask_d), 1, L.ptr(sen_d), L.ptr(ren_d), L.ptr(K_d),
                                               L.ptr(rot), mode, L.ptr(out), n, hw, 0.8, stream), "gdrn_depth_refine_step")
        torch.cuda.synchronize()
        return out.cpu()

    assert torch.equal(run(None, 0), run(R_d, 0))
    got = run(R_d, 1).numpy()
    mn, mx = mask.reshape(n, -1).min(1)[:, None, None], mask.reshape(n, -1).max(1)[:, None, None]
    mask_n = (mask - mn) / (mx - mn)
    sums = []
    for i in range(n):
        x01 = xyz[i].transpose(1, 2, 0)
        w = (R[i] @ x01.reshape(-1, 3).T).T[:, 2].reshape(hw, hw) * mask_n[i] * (ren[i] > 0) * (sensor[i] > 0)
        sums.append(float(w.sum()))
        want = ref_coor_z_step(x01, mask_n[i], sensor[i], ren[i], K[i].astype(np.float64), R[i], t[i].astype(np.float64))
        assert np.abs(got[i] - want).max() < 2e-6, (i, got[i], want)
    assert (np.array([(R[i] @ xyz[i].reshape(3, -1))[2].min() for i in range(3)]) < 0).all()   # negative weights present
    assert sums[0] > 0 and sums[1] < 0 and sums[3] == 0.0
    assert np.array_equal(got[3], t[3]) and not np.array_equal(got[1], t[1])
    with pytest.raises(L.GdrnError):        # coor-z needs the rotations; unknown weight modes are rejected
        run(None, 1)
    with pytest.raises(L.GdrnError):
        run(R_d, 2)


@pytest.mark.gpu
def test_model3d_depth_refine_coor_z_vs_oracle(dev):
    """renderer.depth_refine(coor_z_refine=True): render + coor-z refine, 2 iterations, vs the numpy renderer and the
    reference's coor-z arithmetic; the default weighting is unchanged by the new keyword."""
    from gdrnpp_bop2022_b200.renderer import Model3D, depth_refine, render_depth
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    n = 4
    rs = np.random.RandomState(5)
    v, f = make_icosphere_mesh(3, (0.12, 0.08, 0.1))
    poses, Ks = [], []
    for i in range(n):
        R = _rot(rs.randn(3), rs.rand() * 3)
        poses.append(np.hstack([R, np.array([[rs.randn() * 0.02], [rs.randn() * 0.02], [0.5 + rs.rand() * 0.3]])]))
        Ks.append(np.array([[110.0 + 10 * rs.rand(), 0, 32 + rs.randn()], [0, 112.0, 31 + rs.randn()], [0, 0, 1]]))
    poses, Ks = np.stack(poses).astype(np.float32), np.stack(Ks).astype(np.float32)
    true_poses = poses.copy()
    true_poses[:, :, 3] *= (1 + rs.uniform(-0.04, 0.04, (n, 1)))
    model = Model3D(v, f, device=dev)
    sensor = render_depth(model, torch.from_numpy(true_poses).to(dev), torch.from_numpy(Ks).to(dev), 64, 64)
    xyz = torch.rand(n, 3, 64, 64, generator=torch.Generator().manual_seed(0)).to(dev)
    mask = torch.rand(n, 1, 64, 64, generator=torch.Generator().manual_seed(1)).to(dev)
    rot = torch.from_numpy(poses[:, :, :3]).to(dev).contiguous()
    trans = torch.from_numpy(poses[:, :, 3]).to(dev).contiguous()
    args = (model, rot, trans, torch.from_numpy(Ks).to(dev), xyz, mask, sensor)
    new_t = depth_refine(*args, iters=2, thresh=0.8, coor_z_refine=True).cpu().numpy()
    assert torch.equal(depth_refine(*args, iters=2, thresh=0.8, coor_z_refine=False), depth_refine(*args, iters=2, thresh=0.8))
    mx = mask.view(n, -1).max(1)[0].view(n, 1, 1, 1); mn = mask.view(n, -1).min(1)[0].view(n, 1, 1, 1)
    mnorm = ((mask - mn) / (mx - mn)).cpu().numpy()
    for i in range(n):
        t = poses[i, :, 3].astype(np.float64).copy()
        for _ in range(2):
            ren = OO.render_depth(v, f, np.hstack([poses[i, :, :3], t[:, None]]).astype(np.float32), Ks[i], 64, 64)
            t = ref_coor_z_step(xyz[i].permute(1, 2, 0).cpu().numpy(), mnorm[i, 0], sensor[i].cpu().numpy(), ren, Ks[i].astype(np.float64),
                                poses[i, :, :3], t)
        assert np.abs(new_t[i] - t).max() < 1e-3, i


def _predictor(dev, **kw):
    from gdrnpp_bop2022_b200.predictor import GdrnPredictor
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    objs = {i + 1: "obj_%d" % (i + 1) for i in range(21)}
    extents = {i + 1: np.array([0.1, 0.12, 0.08], np.float32) for i in range(21)}
    return GdrnPredictor(cam=K_CAM.astype(np.float32), objs=objs, extents=extents, state_dict=make_state_dict(), device=dev, **kw)


@pytest.mark.gpu
def test_predictor_pnp_type_and_coor_z(dev, tmp_path):
    """GdrnPredictor honours TEST.PNP_TYPE and TEST.USE_COOR_Z_REFINE from a config file and the pnp_type= /
    use_coor_z_refine= keywords; the default stays pnp_ransac_from_maps bit for bit; an unknown type raises."""
    from gdrnpp_bop2022_b200.pnp_ransac import pnp_net_from_maps, pnp_ransac_from_maps

    rng = np.random.RandomState(11)
    image = rng.randint(0, 256, (480, 640, 3)).astype(np.uint8)
    dets = np.array([[100, 80, 220, 260, 0.9, 0.8, 3], [400, 200, 460, 250, 0.7, 0.9, 10], [300, 100, 380, 190, 0.5, 0.5, 0]], np.float32)

    def run(pred):
        data = pred.preprocessing(dets, image)
        out = pred.inference(data)
        out = {k: v.clone() for k, v in out.items()}
        pred.postprocessing(data, out)
        R = np.stack([r["R"] for r in data["cur_res"]]); t = np.stack([r["t"] for r in data["cur_res"]])
        maps = (out["coor_x"], out["coor_y"], out["coor_z"], out["mask"], data["roi_coord_2d"], data["im_H"], data["im_W"],
                data["roi_extent"], data["cam"])
        return R, t, out, maps

    base = _predictor(dev)
    assert base.cfg.TEST.PNP_TYPE == "ransac_pnp" and base.cfg.TEST.USE_COOR_Z_REFINE is False
    R, t, out, maps = run(base)
    ref = pnp_ransac_from_maps(*maps, mask_thr=base.mask_thr).cpu().numpy()
    assert np.array_equal(R, ref[:, :, :3]) and np.array_equal(t, ref[:, :, 3])
    # config file
    (tmp_path / "cfg.py").write_text(
        "MODEL = dict(PIXEL_MEAN=[0.0, 0.0, 0.0], PIXEL_STD=[255.0, 255.0, 255.0], POSE_NET=dict(NAME='GDRN_double_mask', NUM_CLASSES=21,\n"
        "    OUTPUT_RES=64, BACKBONE=dict(INIT_CFG=dict(type='timm/convnext_base')),\n"
        "    GEO_HEAD=dict(NUM_REGIONS=64, XYZ_CLASS_AWARE=True, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True, MASK_THR_TEST=0.5),\n"
        "    PNP_NET=dict(ROT_TYPE='allo_rot6d', TRANS_TYPE='centroid_z', Z_TYPE='REL')))\n"
        "TEST = dict(USE_PNP=True, PNP_TYPE='net_iter_pnp', USE_DEPTH_REFINE=False, USE_COOR_Z_REFINE=True)\n"
        "INPUT = dict(DZI_PAD_SCALE=1.5, WITH_DEPTH=False)\n")
    pred = _predictor(dev, config_file_path=str(tmp_path / "cfg.py"))
    assert pred.cfg.TEST.PNP_TYPE == "net_iter_pnp" and pred.cfg.TEST.USE_COOR_Z_REFINE is True
    R, t, out, maps = run(pred)
    ref = pnp_net_from_maps(*maps, out["rot"], out["trans"], pnp_type="net_iter_pnp").cpu().numpy()
    assert np.array_equal(R, ref[:, :, :3]) and np.array_equal(t, ref[:, :, 3])
    # keywords override the config
    pred = _predictor(dev, config_file_path=str(tmp_path / "cfg.py"), pnp_type="NET_RANSAC_PNP_ROT", use_coor_z_refine=False)
    assert pred.cfg.TEST.USE_COOR_Z_REFINE is False
    R, t, out, maps = run(pred)
    assert np.array_equal(t, out["trans"].cpu().numpy())         # _rot: the network translation, always
    ref = pnp_net_from_maps(*maps, out["rot"], out["trans"], pnp_type="net_ransac_pnp_rot").cpu().numpy()
    assert np.array_equal(R, ref[:, :, :3])
    with pytest.raises(NotImplementedError):
        _predictor(dev, pnp_type="net_epnp")
