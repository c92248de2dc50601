"""BOP19 pose errors (gdrnpp_bop2022_b200/bop_eval.py, csrc/pose_error.cu).

The numpy restatements below follow lib/pysixd/pose_error.py, misc.py and visibility.py operation for operation; the CPU
tests pin them to tests/golden/ref_pose_error.npz (written by tools/make_golden_pose_error.py from the reference's own
functions) and the GPU tests hold the CUDA kernels to them."""
import json
import os

import numpy as np
import pytest
from scipy import spatial

from gdrnpp_bop2022_b200 import bop_eval

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pose_error.npz")
BOP19_TAUS = list(np.arange(0.05, 0.51, 0.05))


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatements
def dist_im(depth, K):
    """misc.depth_im_to_dist_im_fast with Precomputer's pre_Xs / pre_Ys."""
    xs, ys = np.meshgrid(np.arange(depth.shape[1]), np.arange(depth.shape[0]))
    pre_x = (xs - K[0, 2]) / np.float64(K[0, 0])
    pre_y = (ys - K[1, 2]) / np.float64(K[1, 1])
    return np.sqrt(np.multiply(pre_x, depth) ** 2 + np.multiply(pre_y, depth) ** 2 + depth.astype(np.float64) ** 2)


def visib(d_test, d_model, delta):
    """visibility._estimate_visib_mask, bop19."""
    d_diff = d_model.astype(np.float32) - d_test.astype(np.float32)
    return np.logical_and(np.logical_or(d_diff <= delta, d_test == 0), d_model > 0)


def vsd_np(depth_est, depth_gt, depth_test, K, delta, taus, normalized_by_diameter, diameter):
    dist_test, dist_gt, dist_est = dist_im(depth_test, K), dist_im(depth_gt, K), dist_im(depth_est, K)
    visib_gt = visib(dist_test, dist_gt, delta)
    visib_est = np.logical_or(visib(dist_test, dist_est, delta), np.logical_and(visib_gt, dist_est > 0))
    inter = np.logical_and(visib_gt, visib_est)
    union_count = np.logical_or(visib_gt, visib_est).sum()
    comp_count = union_count - inter.sum()
    dists = np.abs(dist_gt[inter] - dist_est[inter])
    if normalized_by_diameter:
        dists /= diameter
    if union_count == 0:
        return [1.0] * len(taus)
    return [(np.sum(dists >= tau) + comp_count) / float(union_count) for tau in taus]


def transform(pts, R, t):
    return (R.dot(pts.T) + t.reshape((3, 1))).T


def project(pts, K, R, t):
    P = K.dot(np.hstack((R, t.reshape(3, 1))))
    pts_im = P.dot(np.hstack((pts, np.ones((pts.shape[0], 1)))).T)
    pts_im /= pts_im[2, :]
    return pts_im[:2, :].T


def mssd_np(R_e, t_e, R_g, t_g, pts, syms):
    pe = transform(pts, R_e, t_e)
    return min(np.linalg.norm(pe - transform(pts, R_g.dot(s[:, :3]), R_g.dot(s[:, 3:]) + t_g.reshape(3, 1)), axis=1).max()
               for s in syms)


def mspd_np(R_e, t_e, R_g, t_g, K, pts, syms):
    pe = project(pts, K, R_e, t_e)
    return min(np.linalg.norm(pe - project(pts, K, R_g.dot(s[:, :3]), R_g.dot(s[:, 3:]) + t_g.reshape(3, 1)), axis=1).max()
               for s in syms)


def add_np(R_e, t_e, R_g, t_g, pts):
    return np.linalg.norm(transform(pts, R_e, t_e) - transform(pts, R_g, t_g), axis=1).mean()


def adi_np(R_e, t_e, R_g, t_g, pts):
    return spatial.cKDTree(transform(pts, R_e, t_e)).query(transform(pts, R_g, t_g), k=1)[0].mean()


def sym_stack(info, step=0.01):
    return np.stack([np.hstack([s["R"], np.asarray(s["t"], np.float64).reshape(3, 1)])
                     for s in bop_eval.get_symmetry_transformations(info, step)])


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN)
    with open(GOLDEN[:-4] + ".json") as f:
        meta = json.load(f)
    return g, meta


def _golden_vsd_settings(g):
    d = float(g["vsd_diameter"])
    return [(g["vsd_taus_exact"], False), (BOP19_TAUS, True), (g["vsd_taus_exact"] / d, True)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: restatements pinned to the reference fixture
def test_symmetry_transformations_match_reference(golden):
    g, meta = golden
    for name, info in meta["sym_infos"].items():
        ref = g[f"sym_{name}"]
        got = sym_stack(info, meta["max_sym_disc_step"])
        assert got.shape == ref.shape, name
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12, err_msg=name)
    assert len(g["sym_continuous"]) == 314 and len(g["sym_both"]) == 628


def test_point_errors_restatement_matches_reference(golden):
    g, meta = golden
    pts, K = g["pe_pts"], g["pe_K"]
    P = len(g["pe_R_est"])
    args = [(g["pe_R_est"][i], g["pe_t_est"][i], g["pe_R_gt"][i], g["pe_t_gt"][i]) for i in range(P)]
    for name in meta["sym_infos"]:
        syms = g[f"sym_{name}"]
        np.testing.assert_allclose([mssd_np(*a, pts, syms) for a in args], g[f"mssd_{name}"], rtol=1e-12, atol=0)
        np.testing.assert_allclose([mspd_np(*a, K, pts, syms) for a in args], g[f"mspd_{name}"], rtol=1e-12, atol=0)
    np.testing.assert_allclose([add_np(*a, pts) for a in args], g["add"], rtol=1e-12, atol=0)
    np.testing.assert_allclose([adi_np(*a, pts) for a in args], g["adi"], rtol=1e-12, atol=0)


def test_vsd_restatement_matches_reference_exactly(golden):
    g, _ = golden
    errs = g["vsd_errors"]
    d = float(g["vsd_diameter"])
    for si, (taus, normalized) in enumerate(_golden_vsd_settings(g)):
        for ci in range(len(g["vsd_depth_est"])):
            got = vsd_np(g["vsd_depth_est"][ci], g["vsd_depth_gt"][ci], g["vsd_depth_test"][ci], g["vsd_K"], 15, taus,
                         normalized, d)
            assert np.array_equal(np.array(got), errs[si, ci, :len(taus)]), (si, ci)
    # the fixture exercises what it claims: an empty union (1.0), a perfect match (0.0) and partial errors
    assert (errs[1, 2, :] == 1.0).all() and (errs[0, 2, :5] == 1.0).all()
    assert (errs[1, 3, :] == 0.0).all() and errs[0, 3, 0] == 1.0 and 0 < errs[0, 0, 2] < 1   # tau 0: dist 0 >= 0 costs 1


def test_gates_and_symmetric_ids():
    assert bop_eval.sphere_projections_overlap(50.0, [0, 0, 1000.0], [60, 0, 1000.0])
    assert not bop_eval.sphere_projections_overlap(50.0, [0, 0, 1000.0], [120, 0, 1000.0])
    assert not bop_eval.sphere_projections_overlap(50.0, [0, 0, 0.0], [0, 0, 1000.0])
    assert bop_eval.spheres_overlap([0, 0, 1000.0], [0, 0, 1099.0], 100.0)
    assert not bop_eval.spheres_overlap([0, 0, 1000.0], [0, 0, 1100.0], 100.0)
    assert bop_eval.is_symmetric("ycbv", 13, {}) and not bop_eval.is_symmetric("ycbv", 2, {"symmetries_discrete": [1]})
    assert not bop_eval.is_symmetric("other", 2, {"symmetries_continuous": []}) and not bop_eval.is_symmetric("other", 2, {})
    assert bop_eval.is_symmetric("other", 2, {"symmetries_continuous": [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]})


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _surface(rs, H, W, cx, cy, r, z0, sx, sy, noise=2.0):
    yy, xx = np.mgrid[0:H, 0:W]
    d = (z0 + sx * (xx - cx) + sy * (yy - cy) + rs.rand(H, W) * noise).astype(np.float32)
    d[(xx - cx) ** 2 + ((yy - cy) * 1.3) ** 2 > r * r] = 0
    return d


def _vsd_scene(seed=0, H=480, W=640):
    """3 images, 6 GT instances, 8 estimates, 18 pairs: occlusions, missing test depth, empty renders, a gated pair."""
    rs = np.random.RandomState(seed)
    gts = [_surface(rs, H, W, *rs.uniform([150, 120], [490, 360]), rs.uniform(40, 120), rs.uniform(600, 1200),
                    rs.uniform(-1, 1), rs.uniform(-1, 1)) for _ in range(6)]
    ests = [_surface(rs, H, W, *rs.uniform([150, 120], [490, 360]), rs.uniform(40, 120), rs.uniform(600, 1200),
                     rs.uniform(-1, 1), rs.uniform(-1, 1)) for _ in range(6)]
    ests[0] = gts[0].copy()                                       # perfect estimate
    ests[1] = np.where(gts[1] > 0, gts[1] + 12.5, 0).astype(np.float32)   # constant offset along z
    ests.append(np.zeros((H, W), np.float32))                    # empty render (behind the camera)
    ests.append(gts[2].copy())
    tests = []
    for i in range(3):
        scene = np.full((H, W), 1500, np.float32) + rs.rand(H, W).astype(np.float32) * 5
        for gt in gts[2 * i:2 * i + 2]:
            scene = np.where((gt > 0) & (gt < scene), gt + rs.randn(H, W).astype(np.float32), scene)
        scene[rs.rand(H, W) < 0.1] = 0                           # missing depth
        scene[100:180, 200:320] = 400                             # occluder
        tests.append(scene.astype(np.float32))
    pairs = [(e, g, g // 2) for g in range(6) for e in range(8) if (e + g) % 3 == 0 or e == g]
    pairs.append((6, 6 - 1, 2))
    return np.stack(ests), np.stack(gts), np.stack(tests), pairs


@pytest.mark.gpu
@pytest.mark.parametrize("normalized", [True, False])
def test_vsd_gpu_bit_exact_640x480(lib, dev, normalized):
    import torch

    ests, gts, tests, pairs = _vsd_scene()
    P = len(pairs)
    assert P >= 16
    rs = np.random.RandomState(5)
    Ks = np.stack([np.array([[572.4 + i, 0, 325.26 + 0.1 * i], [0, 573.57 - i, 242.05], [0, 0, 1]]) for i in range(P)])
    diam = rs.uniform(80, 200, P)
    gate = np.ones(P, bool)
    gate[3] = False
    # taus placed exactly on the pixel distances of pair 0 (step cost counts dist >= tau)
    e0, g0, _ = pairs[1]
    dg, de = dist_im(gts[g0], Ks[1]), dist_im(ests[e0], Ks[1])
    both = (gts[g0] > 0) & (ests[e0] > 0)
    diffs = np.sort(np.abs(dg[both] - de[both]))
    if normalized:
        taus = list(np.concatenate([BOP19_TAUS, diffs[[len(diffs) // 3, len(diffs) // 2]] / diam[1]]))
    else:
        taus = [0.0, 5.0, 12.5, 20.0, float(diffs[len(diffs) // 3]), float(diffs[len(diffs) // 2]), 80.0]
    pe, pg, pi = (np.array([p[k] for p in pairs], np.int32) for k in range(3))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    got = bop_eval.vsd(T(ests), T(gts), T(tests), T(pe), T(pg), T(pi), T(Ks), T(diam), taus, 15, normalized,
                       gate=T(gate)).cpu().numpy()
    ref = np.array([vsd_np(ests[e], gts[g], tests[i], Ks[p], 15, taus, normalized, diam[p]) if gate[p] else [1.0] * len(taus)
                    for p, (e, g, i) in enumerate(pairs)])
    assert np.array_equal(got, ref), np.argwhere(got != ref)[:10]
    assert (got[pe == 6] == 1.0).all()                              # empty estimate render: union from the GT only
    assert (got[3] == 1.0).all() and got.min() < 0.5 and (got[0] == ref[0]).all()
    again = bop_eval.vsd(T(ests), T(gts), T(tests), T(pe), T(pg), T(pi), T(Ks), T(diam), taus, 15, normalized,
                         gate=T(gate)).cpu().numpy()
    assert np.array_equal(got, again)


@pytest.mark.gpu
def test_vsd_gpu_matches_reference_fixture(lib, dev, golden):
    import torch

    g, _ = golden
    n = len(g["vsd_depth_est"])
    idx = torch.arange(n, dtype=torch.int32, device=dev)
    for si, (taus, normalized) in enumerate(_golden_vsd_settings(g)):
        got = bop_eval.vsd(torch.from_numpy(g["vsd_depth_est"]).to(dev), torch.from_numpy(g["vsd_depth_gt"]).to(dev),
                           torch.from_numpy(g["vsd_depth_test"]).to(dev), idx, idx, idx, torch.from_numpy(g["vsd_K"]),
                           float(g["vsd_diameter"]), taus, 15, normalized).cpu().numpy()
        assert np.array_equal(got, g["vsd_errors"][si, :, :len(taus)]), si


def _rand_rot(rs):
    q = rs.randn(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


SYM_INFOS = {  # 1, 4 and 314 symmetry transforms
    1: {"diameter": 150.0},
    2: {"diameter": 120.0, "symmetries_discrete": [[-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1],
                                                   [1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 3.0, 0, 0, 0, 1],
                                                   [-1, 0, 0, 0, 0, 1, 0, 0, 0, 0, -1, -2.0, 0, 0, 0, 1]]},
    3: {"diameter": 90.0, "symmetries_continuous": [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]},
}


@pytest.mark.gpu
@pytest.mark.parametrize("n_pts", [1, 37, 2048, 20000])
def test_point_errors_gpu_match_restatement(lib, dev, n_pts):
    rs = np.random.RandomState(n_pts)
    points = {o: (rs.rand(n_pts, 3) - 0.5) * np.array([100.0, 70.0, 50.0]) * (0.6 + 0.2 * o) for o in SYM_INFOS}
    models = bop_eval.PoseErrorModels(points, SYM_INFOS, device=dev)
    assert models.n_syms == [1, 4, 314]
    K = np.array([[1066.778, 0, 312.987], [0, 1067.487, 241.311], [0, 0, 1]])
    obj, Re, te, Rg, tg = [], [], [], [], []
    for i in range(12):
        o = 1 + i % 3
        R_g = _rand_rot(rs)
        t_g = np.array([rs.uniform(-100, 100), rs.uniform(-80, 80), rs.uniform(500, 1200)])
        scale = [0.02, 0.2, 1.0][i // 4]
        dR = np.linalg.qr(np.eye(3) + rs.randn(3, 3) * scale)[0]
        dR *= np.sign(np.linalg.det(dR))
        obj.append(o)
        Re.append(dR @ R_g)
        te.append(t_g + rs.randn(3) * [3, 30, 200][i // 4])
        Rg.append(R_g)
        tg.append(t_g)
    P = len(obj)
    gate = np.array([bop_eval.spheres_overlap(te[p], tg[p], SYM_INFOS[obj[p]]["diameter"]) for p in range(P)])
    assert gate.any() and not gate.all()
    syms = {o: sym_stack(SYM_INFOS[o]) for o in SYM_INFOS}
    mssd, mspd = bop_eval.mssd_mspd(models, obj, np.stack(Re), np.stack(te), np.stack(Rg), np.stack(tg), K, gate_mssd=gate)
    use_adi = np.array([o != 1 for o in obj])
    err_ad = bop_eval.ad(models, obj, np.stack(Re), np.stack(te), np.stack(Rg), np.stack(tg), use_adi, gate=gate)
    mssd, mspd, err_ad = mssd.cpu().numpy(), mspd.cpu().numpy(), err_ad.cpu().numpy()
    for p in range(P):
        pts, o = points[obj[p]], obj[p]
        a = (Re[p], te[p], Rg[p], tg[p])
        assert abs(mspd[p] - mspd_np(*a, K, pts, syms[o])) <= 1e-9, p
        if gate[p]:
            assert abs(mssd[p] - mssd_np(*a, pts, syms[o])) <= 1e-9, p
            ref_ad = adi_np(*a, pts) if use_adi[p] else add_np(*a, pts)
            assert abs(err_ad[p] - ref_ad) <= 1e-9, p
        else:
            assert mssd[p] == np.inf and err_ad[p] == np.inf
    # ADD on every pair, ungated, and a second identical call
    add_all = bop_eval.ad(models, obj, np.stack(Re), np.stack(te), np.stack(Rg), np.stack(tg), np.zeros(P, bool))
    np.testing.assert_allclose(add_all.cpu().numpy(), [add_np(Re[p], te[p], Rg[p], tg[p], points[obj[p]]) for p in range(P)],
                               rtol=0, atol=1e-9)
    again = bop_eval.ad(models, obj, np.stack(Re), np.stack(te), np.stack(Rg), np.stack(tg), np.zeros(P, bool))
    assert np.array_equal(add_all.cpu().numpy(), again.cpu().numpy())


@pytest.mark.gpu
def test_point_errors_gpu_match_reference_fixture(lib, dev, golden):
    g, meta = golden
    infos = {i + 1: info for i, info in enumerate(meta["sym_infos"].values())}
    models = bop_eval.PoseErrorModels({o: g["pe_pts"] for o in infos}, infos, meta["max_sym_disc_step"], device=dev)
    P = len(g["pe_R_est"])
    for o, name in zip(infos, meta["sym_infos"]):
        mssd, mspd = bop_eval.mssd_mspd(models, [o] * P, g["pe_R_est"], g["pe_t_est"], g["pe_R_gt"], g["pe_t_gt"], g["pe_K"])
        np.testing.assert_allclose(mssd.cpu().numpy(), g[f"mssd_{name}"], rtol=1e-12, atol=0)
        np.testing.assert_allclose(mspd.cpu().numpy(), g[f"mspd_{name}"], rtol=1e-12, atol=0)
    for flag, key in ((False, "add"), (True, "adi")):
        e = bop_eval.ad(models, [1] * P, g["pe_R_est"], g["pe_t_est"], g["pe_R_gt"], g["pe_t_gt"], [flag] * P)
        np.testing.assert_allclose(e.cpu().numpy(), g[key], rtol=1e-12, atol=0)


@pytest.mark.gpu
def test_bad_inputs_raise(lib, dev):
    import torch

    from gdrnpp_bop2022_b200._lib import GdrnError

    d = torch.zeros((2, 8, 8), dtype=torch.float32)
    K = torch.eye(3, dtype=torch.float64)
    with pytest.raises(GdrnError):
        bop_eval.vsd(d, d, d, [0], [0], [0], K, 1.0, [0.1], 15)
    dc = d.to(dev)
    with pytest.raises(GdrnError):
        bop_eval.vsd(dc, dc[:, :4], dc, [0], [0], [0], K, 1.0, [0.1], 15)
    with pytest.raises(GdrnError):
        bop_eval.vsd(dc, dc, dc, [0, 1], [0], [0], K, 1.0, [0.1], 15)
    with pytest.raises(GdrnError):
        bop_eval.vsd(dc, dc, dc, [2], [0], [0], K, 1.0, [0.1], 15)
    with pytest.raises(GdrnError):
        bop_eval.vsd(dc, dc, dc, [0], [0], [0], K, 1.0, [0.1] * 33, 15)
    models = bop_eval.PoseErrorModels({1: np.zeros((4, 3))}, {1: {"diameter": 1.0}}, device=dev)
    R = np.eye(3)[None]
    with pytest.raises(GdrnError):
        bop_eval.mssd_mspd(models, [2], R, np.zeros((1, 3)), R, np.zeros((1, 3)), np.eye(3))
    with pytest.raises(GdrnError):
        bop_eval.ad(models, [1], R, np.zeros((2, 3)), R, np.zeros((1, 3)), [False])


# ---------------------------------------------------------------------------------------------------------------------
# symmetric objects, matching, scores, signatures, I/O
def test_symmetric_obj_ids_are_the_reference_lists():
    # lib/pysixd/dataset_params.py:98-131 (hope: not defined there)
    ref = {"lm": [3, 7, 10, 11], "lmo": [10, 11], "tless": list(range(1, 31)), "tudl": [],
           "tyol": [3, 4, 5, 6, 7, 8, 10, 11, 12, 13, 15, 16, 17, 18, 19, 21], "ruapc": [8, 9, 12, 13], "icmi": [1, 2, 6],
           "icbin": [1], "itodd": [2, 3, 4, 5, 7, 8, 9, 11, 12, 14, 17, 18, 19, 23, 24, 25, 27, 28],
           "hbs": [10, 12, 18, 29], "hb": [6, 10, 11, 12, 13, 14, 18, 24, 29], "ycbv": [1, 13, 14, 16, 18, 19, 20, 21],
           "ycbvposecnn": [13, 16, 19, 20, 21]}
    assert bop_eval.SYMMETRIC_OBJ_IDS == ref
    sym_info = {"symmetries_discrete": [[1] * 16]}
    assert not bop_eval.is_symmetric("tudl", 1, sym_info) and bop_eval.is_symmetric("icbin", 1, {})


def _canon(x):
    return json.loads(json.dumps(x, sort_keys=True))


def test_matching_scores_and_signatures_match_reference(golden):
    _, meta = golden
    scene_gt = {int(k): v for k, v in meta["scene_gt"].items()}
    valid = {int(k): v for k, v in meta["scene_gt_valid"].items()}
    errs = [{**e, "errors": {int(g): v for g, v in e["errors"].items()}} for e in meta["scene_errs"]]
    for case in meta["matching"]:
        m = bop_eval.match_poses_scene(3, scene_gt, valid, errs, case["th"], case["n_top"])
        assert _canon(m) == case["matches"]
        sc = bop_eval.calc_localization_scores([3, 4], [1, 2, 3], m, case["n_top"])
        assert _canon(sc) == case["scores"]
    sig = meta["signatures"]
    assert [bop_eval.get_error_signature("vsd", -1, vsd_delta=15, vsd_tau=t) for t in bop_eval.VSD_TAUS] \
        + [bop_eval.get_error_signature("vsd", 1, vsd_delta=5, vsd_tau=float("inf")),
           bop_eval.get_error_signature("mssd", -1), bop_eval.get_error_signature("ad", 0)] == sig["error"]
    assert [bop_eval.get_score_signature([th], -1) for th in np.arange(5, 51, 5)] \
        + [bop_eval.get_score_signature([0.02], 0.1), bop_eval.get_score_signature([2, 5], -1)] == sig["score"]


def _box(sx, sy, sz):
    v = np.array([[x, y, z] for x in (-sx, sx) for y in (-sy, sy) for z in (-sz, sz)], np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                  [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int64)
    return v, f


def _write_ply(path, v, f):
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(v), len(f)))
        for p in v:
            fh.write("%r %r %r\n" % tuple(float(c) for c in p))
        for t in f:
            fh.write("3 %d %d %d\n" % tuple(t))


def _write_tree(root, depth_fn=None, n_scenes=3, n_ims=4, seed=3):
    """A tiny BOP tree: ycbv-named dataset, test split, 3 box objects.  depth_fn(scene, im, gts, K) -> [480,640] mm or
    None (a flat depth is written then).  Returns (results rows, scene_gts)."""
    import cv2

    rs = np.random.RandomState(seed)
    base = os.path.join(root, "ycbv")
    os.makedirs(os.path.join(base, "models_eval"))
    sizes = {1: (30.0, 20.0, 15.0), 2: (25.0, 25.0, 40.0), 3: (18.0, 35.0, 22.0)}
    info = {}
    for o, sz in sizes.items():
        v, f = _box(*sz)
        _write_ply(os.path.join(base, "models_eval", "obj_%06d.ply" % o), v, f)
        info[str(o)] = {"diameter": float(2 * np.linalg.norm(sz))}
    info["1"]["symmetries_discrete"] = [[-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]]
    with open(os.path.join(base, "models_eval", "models_info.json"), "w") as fh:
        json.dump(info, fh)
    K = [1066.778, 0, 312.9869, 0, 1067.487, 241.3109, 0, 0, 1]
    targets, rows = [], []
    for s in range(1, n_scenes + 1):
        d = os.path.join(base, "test", "%06d" % s)
        os.makedirs(os.path.join(d, "depth"))
        sg, sc, si = {}, {}, {}
        for im in range(n_ims):
            gts = []
            for o in (1, 2, 3):
                R = _rand_rot(rs)
                t = [rs.uniform(-120, 120), rs.uniform(-90, 90), rs.uniform(700, 1100)]
                gts.append({"obj_id": o, "cam_R_m2c": R.reshape(-1).tolist(), "cam_t_m2c": t})
                targets.append({"scene_id": s, "im_id": im, "obj_id": o, "inst_count": 1})
                kind = (s * 7 + im * 3 + o) % 6
                if kind == 5:
                    continue                                   # missing estimate
                dR = np.linalg.qr(np.eye(3) + rs.randn(3, 3) * (0.02 if kind < 3 else 0.4))[0]
                dR *= np.sign(np.linalg.det(dR))
                te = np.array(t) + rs.randn(3) * (2 if kind < 3 else 40)
                score = 0.5 if kind in (1, 2) else float(rs.rand())   # duplicate scores
                rows.append({"scene_id": s, "im_id": im, "obj_id": o, "score": score, "R": dR @ R, "t": te / 1000.0,
                             "time": 0.25})
                if kind == 2:                                  # a second, worse estimate with the same score
                    rows.append({"scene_id": s, "im_id": im, "obj_id": o, "score": score, "R": R, "t": (te + 30) / 1000.0,
                                 "time": 0.25})
            sg[str(im)] = gts
            sc[str(im)] = {"cam_K": K, "depth_scale": 0.1}
            si[str(im)] = [{"visib_fract": float(v)} for v in rs.rand(3)]
            dep = depth_fn(s, im, gts, np.array(K).reshape(3, 3)) if depth_fn else np.full((480, 640), 900.0)
            cv2.imwrite(os.path.join(d, "depth", "%06d.png" % im), np.round(dep / 0.1).astype(np.uint16))
        for name, obj in (("scene_gt.json", sg), ("scene_camera.json", sc), ("scene_gt_info.json", si)):
            with open(os.path.join(d, name), "w") as fh:
                json.dump(obj, fh)
    with open(os.path.join(base, "test_targets_bop19.json"), "w") as fh:
        json.dump(targets, fh)
    return rows


def test_loaders_and_cli_parsing(tmp_path):
    rows = _write_tree(str(tmp_path))
    ds = bop_eval.BopSplit(str(tmp_path), "ycbv", "test")
    assert ds.scene_ids == [1, 2, 3] and ds.im_size == (640, 480)
    gt = bop_eval.load_scene_gt(ds.scene_file(1, "scene_gt.json"))
    cam = bop_eval.load_scene_camera(ds.scene_file(1, "scene_camera.json"))
    assert gt[0][0]["cam_R_m2c"].shape == (3, 3) and gt[0][0]["cam_t_m2c"].shape == (3, 1) and cam[0]["cam_K"][0, 0] == 1066.778
    d = ds.depth(1, 0, 0.1)
    assert d.dtype == np.float32 and d.shape == (480, 640) and d[0, 0] == np.float32(9000) * np.float32(0.1)
    assert sorted(ds.models_info()) == [1, 2, 3] and ds.model(2)["faces"].shape == (12, 3)
    csv = str(tmp_path / "m_ycbv-test.csv")
    bop_eval.write_bop_results_csv(rows, csv)
    ests = bop_eval.load_bop_results(csv)
    assert len(ests) == len(rows)
    np.testing.assert_allclose(ests[3]["t"].ravel(), rows[3]["t"] * 1000, rtol=1e-15)
    assert np.array_equal(ests[3]["R"], rows[3]["R"]) and ests[3]["score"] == rows[3]["score"]
    a = bop_eval.parse_args(["--results_path", str(tmp_path), "--result_filenames", "m_ycbv-test.csv", "--renderer_type",
                             "egl", "--error_types", "vsd,mssd,mspd,ad", "--eval_path", str(tmp_path / "ev"),
                             "--targets_filename", "test_targets_bop19.json", "--n_top", "-1", "--score_only"])
    assert a.error_types == ["vsd", "mssd", "mspd", "ad"] and a.score_only and a.n_top == -1
    with pytest.raises(SystemExit):
        bop_eval.parse_args(["--result_filenames", "x.csv", "--error_types", "mssd,reS"])


@pytest.mark.gpu
def test_evaluate_synthetic_dataset_matches_host_and_cli(lib, dev, tmp_path):
    import subprocess
    import sys

    import torch

    holder = {}

    def scene_depth(s, im, gts, K):
        m = holder["meshes"]
        d = m.render([g["obj_id"] for g in gts], np.stack([np.reshape(g["cam_R_m2c"], (3, 3)) for g in gts]),
                     np.stack([g["cam_t_m2c"] for g in gts]), np.stack([K] * len(gts)), 480, 640).cpu().numpy()
        d = np.where(d > 0, d, np.inf).min(0)
        d[~np.isfinite(d)] = 1500
        rs = np.random.RandomState(s * 10 + im)
        d[rs.rand(480, 640) < 0.05] = 0                     # holes
        d[200:260, 280:400] = np.minimum(d[200:260, 280:400], 650)   # occluder
        return d

    ply_meshes = {o: _box(*sz) for o, sz in {1: (30.0, 20.0, 15.0), 2: (25.0, 25.0, 40.0), 3: (18.0, 35.0, 22.0)}.items()}
    holder["meshes"] = bop_eval.VsdMeshes(ply_meshes, device=dev)
    rows = _write_tree(str(tmp_path), scene_depth)
    res = tmp_path / "res"
    res.mkdir()
    bop_eval.write_bop_results_csv(rows, str(res / "m_ycbv-test.csv"))
    ds = bop_eval.BopSplit(str(tmp_path), "ycbv", "test")
    ests = bop_eval.load_bop_results(str(res / "m_ycbv-test.csv"))
    targets = bop_eval.load_json(os.path.join(ds.base_path, "test_targets_bop19.json"))
    sids = [1, 2, 3]
    sgt = {s: bop_eval.load_scene_gt(ds.scene_file(s, "scene_gt.json")) for s in sids}
    scam = {s: bop_eval.load_scene_camera(ds.scene_file(s, "scene_camera.json")) for s in sids}
    sinfo = {s: bop_eval.load_json(ds.scene_file(s, "scene_gt_info.json"), keys_to_int=True) for s in sids}
    minfo = ds.models_info()
    plys = {o: ds.model(o) for o in minfo}
    models = bop_eval.PoseErrorModels({o: m["pts"] for o, m in plys.items()}, minfo, device=dev)
    meshes = bop_eval.VsdMeshes({o: (m["pts"], m["faces"]) for o, m in plys.items()}, device=dev)
    depth = lambda s, i: ds.depth(s, i, 0.1)  # noqa: E731
    types = ["vsd", "mssd", "mspd", "ad"]
    final, errors = bop_eval.evaluate(types, "ycbv", ests, targets, sgt, scam, sinfo, minfo, 640, models, meshes, depth,
                                      scene_ids=ds.scene_ids)
    final2, errors2 = bop_eval.evaluate(types, "ycbv", ests, targets, sgt, scam, sinfo, minfo, 640, models, meshes, depth,
                                        scene_ids=ds.scene_ids)
    assert final == final2 and errors == errors2
    assert 0 < final["bop19_average_recall"] < 1
    # chunking changes no bit
    one = bop_eval.calc_errors("vsd", "ycbv", ests, targets, sgt, scam, minfo, meshes=meshes, load_depth=depth,
                               vsd_delta=15, max_bytes=1)
    assert one == errors["vsd"]
    # host restatement of every error, VSD on the library's own renders; the same matching / scoring
    org = {}
    for e in ests:
        org.setdefault((e["scene_id"], e["im_id"], e["obj_id"]), []).append(e)
    syms = {o: sym_stack(minfo[o]) for o in minfo}
    host = {}
    for et in types:
        host[et] = {}
        for s, recs in errors[et].items():
            host[et][s] = []
            for r in recs:
                est = org[(s, r["im_id"], r["obj_id"])][r["est_id"]]
                K = scam[s][r["im_id"]]["cam_K"]
                o, d = r["obj_id"], minfo[r["obj_id"]]["diameter"]
                pts = plys[o]["pts"]
                he = {}
                for g in r["errors"]:
                    gt = sgt[s][r["im_id"]][g]
                    a = (est["R"], est["t"], gt["cam_R_m2c"], gt["cam_t_m2c"])
                    if et == "vsd":
                        if not bop_eval.sphere_projections_overlap(0.5 * d, est["t"], gt["cam_t_m2c"]):
                            he[g] = [1.0] * 10
                            continue
                        de = meshes.render([o], est["R"][None], est["t"].reshape(1, 3), K[None], 480, 640)[0].cpu().numpy()
                        dg = meshes.render([o], gt["cam_R_m2c"][None], gt["cam_t_m2c"].reshape(1, 3), K[None], 480,
                                           640)[0].cpu().numpy()
                        he[g] = [float(v) for v in vsd_np(de, dg, depth(s, r["im_id"]), K, 15, bop_eval.VSD_TAUS, True, d)]
                    elif et == "mspd":
                        he[g] = [mspd_np(*a, K, pts, syms[o])]
                    elif not bop_eval.spheres_overlap(est["t"], gt["cam_t_m2c"], d):
                        he[g] = [float("inf")]
                    elif et == "mssd":
                        he[g] = [mssd_np(*a, pts, syms[o])]
                    else:
                        he[g] = [adi_np(*a, pts) if o == 1 else add_np(*a, pts)]
                host[et][s].append({**r, "errors": he})
        if et == "vsd":
            assert host[et] == errors[et]
        ar = bop_eval.average_recalls(et, host[et], targets, sgt, sinfo, minfo, 640, scene_ids=ds.scene_ids)[0]
        assert ar == final["bop19_average_recall_" + et], et
    # the script, run by path, writes the same ARs
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "gdrnpp_bop2022_b200", "bop_eval.py"), "--results_path=" + str(res),
           "--result_filenames=m_ycbv-test.csv", "--renderer_type=egl", "--error_types=vsd,mssd,mspd,ad",
           "--eval_path=" + str(tmp_path / "ev"), "--targets_filename=test_targets_bop19.json", "--n_top=-1",
           "--datasets_path=" + str(tmp_path)]
    for extra in ([], ["--score_only"]):
        subprocess.run(cmd + extra, check=True, cwd=str(tmp_path))
        got = bop_eval.load_json(str(tmp_path / "ev" / "m_ycbv-test" / "scores_bop19.json"))
        for k, v in final.items():
            assert got[k] == float(v), (k, extra)
        assert got["bop19_average_time_per_image"] == 0.25
    assert os.path.exists(tmp_path / "ev" / "m_ycbv-test" / "error:vsd_ntop:-1_delta:15.000_tau:0.050" / "errors_000001.json")
