"""Every error type of eval_pose_results_more.py (gdrnpp_bop2022_b200/eval_pose_results_more.py, bop_eval.rt_errors /
proj_errors, csrc/pose_error.cu sym_rt_kernel / sym_proj_mean_kernel).

The numpy restatements below follow lib/pysixd/pose_error.py operation for operation; the CPU tests pin them to
tests/golden/ref_pose_error_more.npz (written by tools/make_golden_pose_error_more.py from the reference's own functions
and scripts) and the GPU tests hold the CUDA kernels to them."""
import filecmp
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from gdrnpp_bop2022_b200 import bop_eval
from gdrnpp_bop2022_b200 import eval_pose_results_more as more
from test_bop_eval import _box, _rand_rot, _write_tree, add_np, adi_np, sym_stack

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pose_error_more.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatements (syms: [S,3,4] stacks of [R|t])
def re_np(R_e, R_g):
    trace = np.trace(np.dot(R_e, R_g.T))
    trace = trace if trace <= 3 else 3
    return np.rad2deg(np.arccos(min(1.0, max(-1.0, 0.5 * (trace - 1.0)))))


def re_sym_np(R_e, R_g, syms):
    return min(re_np(R_e, R_g.dot(s[:, :3])) for s in syms)


def te_np(t_e, t_g):
    return np.linalg.norm(np.ravel(t_g) - np.ravel(t_e))


def te_sym_np(t_e, t_g, R_g, syms):
    return min(np.linalg.norm(R_g.dot(s[:, 3:]).reshape(3) + np.ravel(t_g) - np.ravel(t_e)) for s in syms)


def transform_2d(pts, R, t, K):
    c = K.dot(R.dot(pts.T) + np.reshape(t, (3, 1)))
    return np.stack([c[0, :] / c[2, :], c[1, :] / c[2, :]], axis=1)


def arp_2d_np(R_e, t_e, R_g, t_g, pts, K):
    return np.linalg.norm(transform_2d(pts, R_e, t_e, K) - transform_2d(pts, R_g, t_g, K), axis=1).mean()


def arp_2d_sym_np(R_e, t_e, R_g, t_g, pts, K, syms):
    pe = transform_2d(pts, R_e, t_e, K)
    return min(np.linalg.norm(pe - transform_2d(pts, R_g.dot(s[:, :3]), R_g.dot(s[:, 3:]) + np.reshape(t_g, (3, 1)), K),
                              axis=1).mean() for s in syms)


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN)
    with open(GOLDEN[:-4] + ".json") as f:
        meta = json.load(f)
    return g, meta


def _golden_pairs(g):
    return [(g["R_est"][i], g["t_est"][i], g["R_gt"][i], g["t_gt"][i]) for i in range(len(g["R_est"]))]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
def test_restatements_match_reference(golden):
    g, meta = golden
    pts, K = g["pts"], g["K"]
    a = _golden_pairs(g)
    close = lambda got, key: np.testing.assert_allclose(got, g[key], rtol=1e-12, atol=0, err_msg=key)  # noqa: E731
    close([re_np(x[0], x[2]) for x in a], "re")
    close([te_np(x[1], x[3]) for x in a], "te")
    close([arp_2d_np(*x, pts, K) for x in a], "arp_2d")
    close([add_np(*x, pts) for x in a], "add")
    close([adi_np(*x, pts) for x in a], "adi")
    for name in meta["sym_infos"]:
        syms = g[f"sym_{name}"]
        close([re_sym_np(x[0], x[2], syms) for x in a], f"re_sym_{name}")
        close([te_sym_np(x[1], x[3], x[2], syms) for x in a], f"te_sym_{name}")
        close([arp_2d_sym_np(*x, pts, K, syms) for x in a], f"arp_2d_sym_{name}")
    cases = meta["cases"]
    assert g["re"][cases.index("identity")] == 0.0 and g["re"][cases.index("rot180")] == 180.0
    assert abs(g["re"][cases.index("small_angle")] - np.rad2deg(1e-4)) < 1e-9
    assert g["te"][cases.index("off_1m")] == 1000.0 and np.isfinite(g["arp_2d"]).all()


def test_continuous_symmetry_sets_hold_no_identity(golden):
    g, meta = golden
    ident = np.hstack([np.eye(3), np.zeros((3, 1))])
    dist = {name: np.abs(g[f"sym_{name}"] - ident).max(axis=(1, 2)).min() for name in meta["sym_infos"]}
    assert dist["none"] == 0.0 and dist["discrete"] == 0.0
    assert dist["continuous"] > 1e-3 and dist["both"] > 1e-3
    for name in meta["sym_infos"]:   # restated by bop_eval exactly
        np.testing.assert_allclose(sym_stack(meta["sym_infos"][name], meta["max_sym_disc_step"]), g[f"sym_{name}"],
                                   rtol=0, atol=1e-12)
    # so re / te / proj differ from their symmetric forms even for a perfect estimate
    i = meta["cases"].index("identity")
    assert g["re"][i] == 0.0 and g["re_sym_continuous"][i] > 1.0 and g["arp_2d_sym_continuous"][i] > 0.0


def test_tables_are_the_reference_tables(golden):
    _, meta = golden
    assert list(more.KNOWN_ERROR_TYPES) == [e["type"] for e in meta["errors"]]
    for e in meta["errors"]:
        assert [[float(t) for t in th] for th in more.CORRECT_TH[e["type"]]] == e["correct_th"], e["type"]
        assert e["n_top"] == -1
    assert more.DEFAULT_ERROR_TYPES == meta["default_error_types"]
    assert list(bop_eval.NORMALIZED_BY_DIAMETER) == meta["normalized_by_diameter"]
    assert list(bop_eval.NORMALIZED_BY_IM_WIDTH) == meta["normalized_by_im_width"]


def test_parse_args():
    for types in ("mspd,mssd,vsd,ad,reS,teS", "ad,rete,re,te,proj", ",".join(more.KNOWN_ERROR_TYPES)):
        a = more.parse_args(["--result_filenames", "m_ycbv-test.csv", "--error_types", types, "--datasets_path", "/d"])
        assert a.error_types == types.split(",") and a.datasets_path == "/d"
    assert more.parse_args(["--result_filenames", "x.csv"]).error_types == "mspd,mssd,vsd,reteS,add,adi,teS,reS,projS".split(",")
    for bad in ("cus", "foo", "vsd,cus"):
        with pytest.raises(SystemExit):
            more.parse_args(["--result_filenames", "x.csv", "--error_types", bad])
    with pytest.raises(ValueError):
        more.calc_errors("cus", "ycbv", [], [], {}, {}, {})


def test_two_component_scoring():
    """rete: a match needs both components below their thresholds, greedy in the reference's GT order."""
    assert bop_eval.get_score_signature(more.CORRECT_TH["rete"][0], -1) == "th:2.000-2.000_min-visib:-1.000"
    scene_gt = {0: [{"obj_id": 1}, {"obj_id": 1}, {"obj_id": 2}]}
    targets = [{"scene_id": 1, "im_id": 0, "obj_id": 1, "inst_count": 2},
               {"scene_id": 1, "im_id": 0, "obj_id": 2, "inst_count": 1}]
    infos = {1: {0: [{"visib_fract": 0.5}] * 3}}
    errs = {1: [{"im_id": 0, "obj_id": 1, "est_id": 0, "score": 0.9, "errors": {0: [1.0, 1.9], 1: [0.5, 1.95]}},
                {"im_id": 0, "obj_id": 1, "est_id": 1, "score": 0.8, "errors": {0: [0.1, 0.1], 1: [1.99, 3.0]}},
                {"im_id": 0, "obj_id": 2, "est_id": 0, "score": 0.7, "errors": {2: [2.5, 0.5]}}]}
    models_info = {1: {"diameter": 10.0}, 2: {"diameter": 10.0}}
    sc, m = bop_eval.calc_scores("rete", errs, targets, {1: scene_gt}, infos, models_info, 640, [2, 2], -1)
    assert sc["recall"] == pytest.approx(1 / 3) and sc["tp_count"] == 1
    assert [(x["gt_id"], x["est_id"]) for x in m] == [(0, 0), (1, -1), (2, -1)]
    assert m[0]["error"] == [1.0, 1.9] and m[0]["error_norm"] == [0.5, 0.95]   # not normalised by the diameter
    sc, m = bop_eval.calc_scores("rete", errs, targets, {1: scene_gt}, infos, models_info, 640, [5, 5], -1)
    assert sc["recall"] == 1.0 and [(x["gt_id"], x["est_id"]) for x in m] == [(0, 0), (1, 1), (2, 0)]


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _sym_infos(golden):
    _, meta = golden
    return {i + 1: info for i, info in enumerate(meta["sym_infos"].values())}   # 1, 3, 314 and 628 transforms


def _special_pairs(rs, n_random):
    """(R_e, t_e, R_g, t_g): random perturbations, an exact identity, 180 degrees and 1e-4 rad."""
    out = []
    for i in range(n_random):
        R_g = _rand_rot(rs)
        t_g = np.array([rs.uniform(-100, 100), rs.uniform(-80, 80), rs.uniform(500, 1200)])
        dR = np.linalg.qr(np.eye(3) + rs.randn(3, 3) * [0.02, 0.3][i % 2])[0]
        dR *= np.sign(np.linalg.det(dR))
        out.append((dR @ R_g, t_g + rs.randn(3) * [3, 40][i % 2], R_g, t_g))
    R_g, t_g = _rand_rot(rs), np.array([10.0, -20.0, 900.0])
    flip = np.diag([-1.0, -1.0, 1.0])
    c, s = np.cos(1e-4), np.sin(1e-4)
    small = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    out += [(R_g.copy(), t_g.copy(), R_g, t_g), (R_g @ flip, t_g + [2.0, 0, 0], R_g, t_g),
            (small @ R_g, t_g + [0.01, 0, 0], R_g, t_g)]
    return out


def _check_against_restatement(models, points, syms, obj, Re, te, Rg, tg, K):
    P = len(obj)
    for use in (False, True):
        re_d, te_mm = (x.cpu().numpy() for x in bop_eval.rt_errors(models, obj, Re, te, Rg, tg, use))
        pr = bop_eval.proj_errors(models, obj, Re, te, Rg, tg, K, use).cpu().numpy()
        for p in range(P):
            o = obj[p]
            a = (Re[p], te[p], Rg[p], tg[p])
            if use:
                ref = (re_sym_np(Re[p], Rg[p], syms[o]), te_sym_np(te[p], tg[p], Rg[p], syms[o]),
                       arp_2d_sym_np(*a, points[o], K, syms[o]))
            else:
                ref = (re_np(Re[p], Rg[p]), te_np(te[p], tg[p]), arp_2d_np(*a, points[o], K))
            assert abs(re_d[p] - ref[0]) <= 1e-5, (use, p, re_d[p], ref[0])
            assert abs(te_mm[p] - ref[1]) <= 1e-9 * abs(ref[1]), (use, p, te_mm[p], ref[1])
            assert abs(pr[p] - ref[2]) <= 1e-9 * abs(ref[2]), (use, p, pr[p], ref[2])
    return re_d, te_mm, pr


@pytest.mark.gpu
@pytest.mark.parametrize("n_pts", [1, 37, 2048, 20000])
def test_rt_proj_gpu_match_restatement(lib, dev, golden, n_pts):
    infos = _sym_infos(golden)
    rs = np.random.RandomState(n_pts)
    points = {o: (rs.rand(n_pts, 3) - 0.5) * np.array([100.0, 70.0, 50.0]) * (0.6 + 0.2 * o) for o in infos}
    models = bop_eval.PoseErrorModels(points, infos, device=dev)
    assert models.n_syms == [1, 3, 314, 628]
    K = np.array([[1066.778, 0, 312.987], [0, 1067.487, 241.311], [0, 0, 1]])
    obj, pairs = [], []
    for o in infos:
        ps = _special_pairs(rs, 3)
        obj += [o] * len(ps)
        pairs += ps
    Re, te, Rg, tg = (np.stack([p[k] for p in pairs]) for k in range(4))
    syms = {o: sym_stack(infos[o]) for o in infos}
    re_s, te_s, pr_s = _check_against_restatement(models, points, syms, obj, Re, te, Rg, tg, K)
    ident = [i for i in range(len(obj)) if np.array_equal(Re[i], Rg[i]) and np.array_equal(te[i], tg[i])]
    re_i, te_i = (x.cpu().numpy() for x in bop_eval.rt_errors(models, obj, Re, te, Rg, tg, False))
    assert (re_i[ident] < 1e-5).all() and (te_i[ident] == 0.0).all()
    assert (bop_eval.proj_errors(models, obj, Re, te, Rg, tg, K, False).cpu().numpy()[ident] == 0.0).all()
    # the continuous sets hold no identity: a perfect estimate of a continuously symmetric object has a symmetric error
    assert all(re_s[i] > 0.5 for i in ident if obj[i] in (3, 4))


@pytest.mark.gpu
def test_rt_proj_gpu_match_reference_fixture(lib, dev, golden):
    g, meta = golden
    infos = _sym_infos(golden)
    models = bop_eval.PoseErrorModels({o: g["pts"] for o in infos}, infos, meta["max_sym_disc_step"], device=dev)
    P = len(g["R_est"])
    args = (g["R_est"], g["t_est"], g["R_gt"], g["t_gt"])
    for o, name in zip(infos, meta["sym_infos"]):
        for use, keys in ((False, ("re", "te", "arp_2d")), (True, (f"re_sym_{name}", f"te_sym_{name}", f"arp_2d_sym_{name}"))):
            re_d, te_mm = (x.cpu().numpy() for x in bop_eval.rt_errors(models, [o] * P, *args, use))
            pr = bop_eval.proj_errors(models, [o] * P, *args, g["K"], use).cpu().numpy()
            np.testing.assert_allclose(re_d, g[keys[0]], rtol=0, atol=1e-5, err_msg=keys[0])
            np.testing.assert_allclose(te_mm, g[keys[1]], rtol=1e-9, atol=0, err_msg=keys[1])
            np.testing.assert_allclose(pr, g[keys[2]], rtol=1e-9, atol=0, err_msg=keys[2])
    for use_adi, key in ((False, "add"), (True, "adi")):   # ABS* / AUC*: ADD / ADI with no gate
        e = bop_eval.ad(models, [1] * P, *args, [use_adi] * P).cpu().numpy()
        np.testing.assert_allclose(e, g[key], rtol=1e-9, atol=0, err_msg=key)


@pytest.mark.gpu
def test_rt_proj_gpu_bits_do_not_depend_on_batching(lib, dev, golden):
    infos = _sym_infos(golden)
    rs = np.random.RandomState(11)
    points = {o: (rs.rand(3000 + 77 * o, 3) - 0.5) * 90.0 for o in infos}
    models = bop_eval.PoseErrorModels(points, infos, device=dev)
    K = np.array([[600.0, 0, 320.5], [0, 610.0, 240.5], [0, 0, 1]])
    pairs = _special_pairs(rs, 9)
    obj = [1 + i % 4 for i in range(len(pairs))]
    use = np.array([i % 3 != 0 for i in range(len(pairs))])
    Re, te, Rg, tg = (np.stack([p[k] for p in pairs]) for k in range(4))

    def run(sel):
        r, t = bop_eval.rt_errors(models, [obj[i] for i in sel], Re[sel], te[sel], Rg[sel], tg[sel], use[sel])
        pr = bop_eval.proj_errors(models, [obj[i] for i in sel], Re[sel], te[sel], Rg[sel], tg[sel], K, use[sel])
        return np.stack([r.cpu().numpy(), t.cpu().numpy(), pr.cpu().numpy()])

    all_ = np.arange(len(obj))
    first = run(all_)
    assert np.array_equal(first, run(all_))
    one_by_one = np.concatenate([run(np.array([i])) for i in all_], axis=1)
    assert np.array_equal(first, one_by_one)
    assert np.array_equal(first[:, ::-1], run(all_[::-1]))


@pytest.mark.gpu
def test_rt_proj_bad_inputs_raise(lib, dev):
    import torch

    from gdrnpp_bop2022_b200._lib import GdrnError

    models = bop_eval.PoseErrorModels({1: np.zeros((4, 3))}, {1: {"diameter": 1.0}}, device=dev)
    R, t, K = np.eye(3)[None], np.zeros((1, 3)), np.eye(3)
    r, tt = bop_eval.rt_errors(models, [], R[:0], t[:0], R[:0], t[:0], True)
    assert r.shape == (0,) and tt.shape == (0,) and r.is_cuda and r.dtype == torch.float64
    assert bop_eval.proj_errors(models, [], R[:0], t[:0], R[:0], t[:0], K, True).shape == (0,)
    bad = [dict(obj=[2]), dict(t=np.zeros((2, 3))), dict(R=np.eye(4)[None]), dict(use=[True, False]),
           dict(R=torch.eye(3)[None].double()), dict(K=torch.eye(3).double())]
    for b in bad:
        args = (models, b.get("obj", [1]), b.get("R", R), b.get("t", t), R, t)
        with pytest.raises(GdrnError):
            bop_eval.proj_errors(*args, b.get("K", K), b.get("use", True))
        if "K" not in b:
            with pytest.raises(GdrnError):
                bop_eval.rt_errors(*args, b.get("use", True))
    cpu_models = bop_eval.PoseErrorModels({1: np.zeros((4, 3))}, {1: {"diameter": 1.0}}, device="cpu")
    with pytest.raises(GdrnError):
        bop_eval.rt_errors(cpu_models, [1], R, t, R, t, True)
    with pytest.raises(GdrnError):
        bop_eval.proj_errors(cpu_models, [1], R, t, R, t, K, True)


def _host_error(et, est, gt, K, pts, syms, symmetric):
    a = (est["R"], est["t"], gt["cam_R_m2c"], gt["cam_t_m2c"])
    base, use = et.rstrip("S"), et.endswith("S")
    r = re_sym_np(a[0], a[2], syms) if use else re_np(a[0], a[2])
    t = (te_sym_np(a[1], a[3], a[2], syms) if use else te_np(a[1], a[3])) / 10
    if base in ("re", "te", "rete"):
        return {"re": [r], "te": [t], "rete": [r, t]}[base]
    if base == "proj":
        return [arp_2d_sym_np(*a, pts, K, syms) if use else arp_2d_np(*a, pts, K)]
    kind = et[3:]
    return [(adi_np(*a, pts) if kind == "adi" or (kind == "ad" and symmetric) else add_np(*a, pts)) / 10]


@pytest.mark.gpu
def test_evaluate_every_error_type_synthetic_dataset(lib, dev, tmp_path):
    holder = {}

    def scene_depth(s, im, gts, K):
        d = holder["meshes"].render([g["obj_id"] for g in gts], np.stack([np.reshape(g["cam_R_m2c"], (3, 3)) for g in gts]),
                                    np.stack([g["cam_t_m2c"] for g in gts]), np.stack([K] * len(gts)), 480, 640).cpu().numpy()
        d = np.where(d > 0, d, np.inf).min(0)
        d[~np.isfinite(d)] = 1500
        d[np.random.RandomState(s * 10 + im).rand(480, 640) < 0.05] = 0
        return d

    sizes = {1: (30.0, 20.0, 15.0), 2: (25.0, 25.0, 40.0), 3: (18.0, 35.0, 22.0)}
    holder["meshes"] = bop_eval.VsdMeshes({o: _box(*sz) for o, sz in sizes.items()}, device=dev)
    rows = _write_tree(str(tmp_path), scene_depth)
    keys = [(r["scene_id"], r["im_id"], r["obj_id"]) for r in rows]
    far = next(i for i, k in enumerate(keys) if keys.count(k) == 1)
    rows[far]["t"] = rows[far]["t"] + np.array([0.0, 0.0, 1.0])   # 1 m off: ad is inf, ABSad is not
    res = tmp_path / "res"
    res.mkdir()
    bop_eval.write_bop_results_csv(rows, str(res / "m_ycbv-test.csv"))
    ds = bop_eval.BopSplit(str(tmp_path), "ycbv", "test")
    ests = bop_eval.load_bop_results(str(res / "m_ycbv-test.csv"))
    targets = bop_eval.load_json(os.path.join(ds.base_path, "test_targets_bop19.json"))
    sgt = {s: bop_eval.load_scene_gt(ds.scene_file(s, "scene_gt.json")) for s in ds.scene_ids}
    scam = {s: bop_eval.load_scene_camera(ds.scene_file(s, "scene_camera.json")) for s in ds.scene_ids}
    sinfo = {s: bop_eval.load_json(ds.scene_file(s, "scene_gt_info.json"), keys_to_int=True) for s in ds.scene_ids}
    minfo = ds.models_info()
    plys = {o: ds.model(o) for o in minfo}
    models = bop_eval.PoseErrorModels({o: m["pts"] for o, m in plys.items()}, minfo, device=dev)
    meshes = bop_eval.VsdMeshes({o: (m["pts"], m["faces"]) for o, m in plys.items()}, device=dev)
    depth = lambda s, i: ds.depth(s, i, 0.1)  # noqa: E731
    final, errors = more.evaluate(list(more.KNOWN_ERROR_TYPES), "ycbv", ests, targets, sgt, scam, sinfo, minfo, 640, models,
                                  meshes, depth, scene_ids=ds.scene_ids)
    assert sorted(final) == sorted(["bop19_average_recall_" + t for t in more.KNOWN_ERROR_TYPES] + ["bop19_average_recall"])
    # the BOP19 types are bop_eval's own
    bop19 = list(bop_eval.ERROR_TYPES)
    final19, errors19 = bop_eval.evaluate(bop19, "ycbv", ests, targets, sgt, scam, sinfo, minfo, 640, models, meshes, depth,
                                          scene_ids=ds.scene_ids)
    assert all(errors[t] == errors19[t] and final["bop19_average_recall_" + t] == final19["bop19_average_recall_" + t]
               for t in bop19) and final["bop19_average_recall"] == final19["bop19_average_recall"]
    # every other type: host-restated errors through the same scoring give the same AR
    org = {}
    for e in ests:
        org.setdefault((e["scene_id"], e["im_id"], e["obj_id"]), []).append(e)
    syms = {o: sym_stack(minfo[o]) for o in minfo}
    for et in more.KNOWN_ERROR_TYPES:
        if et in bop19:
            continue
        host = {}
        for s, recs in errors[et].items():
            host[s] = []
            for r in recs:
                est = org[(s, r["im_id"], r["obj_id"])][r["est_id"]]
                o = r["obj_id"]
                he = {g: _host_error(et, est, sgt[s][r["im_id"]][g], scam[s][r["im_id"]]["cam_K"], plys[o]["pts"], syms[o],
                                     bop_eval.is_symmetric("ycbv", o, minfo[o])) for g in r["errors"]}
                for g, v in he.items():
                    got = r["errors"][g]
                    assert len(got) == len(v) and np.isfinite(got).all(), (et, g)
                    tol = [1e-5] * len(v) if et.startswith("re") else [1e-9 * abs(x) for x in v]
                    if et.startswith("rete"):
                        tol = [1e-5, 1e-9 * abs(v[1])]
                    assert all(abs(x - y) <= tt for x, y, tt in zip(got, v, tol)), (et, got, v)
                host[s].append({**r, "errors": he})
        ar = bop_eval.average_recalls(et, host, targets, sgt, sinfo, minfo, 640, scene_ids=ds.scene_ids,
                                      correct_th=more.CORRECT_TH)[0]
        assert ar == final["bop19_average_recall_" + et], et
    # the far-off estimate: ad is gated to inf, ABSad / AUCad are finite (in cm)
    fs, fi, fo = keys[far]
    rec = lambda et: next(r for r in errors[et][fs] if r["im_id"] == fi and r["obj_id"] == fo)  # noqa: E731
    assert all(v == [float("inf")] for v in rec("ad")["errors"].values())
    assert all(90 < v[0] < 200 for v in rec("ABSad")["errors"].values()) and rec("AUCad") == rec("ABSad")
    assert 0 < final["bop19_average_recall_ABSad"] <= 1

    # by path: the six error types of most shipped configs, and --score_only reproduces the scores
    def cli(script, types, ev, extra=()):
        cmd = [sys.executable, os.path.join(ROOT, "gdrnpp_bop2022_b200", script), "--results_path=" + str(res),
               "--result_filenames=m_ycbv-test.csv", "--renderer_type=egl", "--error_types=" + types,
               "--eval_path=" + str(tmp_path / ev), "--targets_filename=test_targets_bop19.json", "--n_top=-1",
               "--datasets_path=" + str(tmp_path)] + list(extra)
        subprocess.run(cmd, check=True, cwd=str(tmp_path))
        return tmp_path / ev / "m_ycbv-test"

    six = ["mspd", "mssd", "vsd", "ad", "reS", "teS"]
    out = cli("eval_pose_results_more.py", ",".join(six), "ev6")
    first = (out / "scores_bop19.json").read_bytes()
    got = json.loads(first)
    assert sorted(got) == sorted(["bop19_average_recall_" + t for t in six] + ["bop19_average_recall",
                                                                              "bop19_average_time_per_image"])
    for k, v in got.items():
        assert v == (0.25 if k == "bop19_average_time_per_image" else float(final[k])), k
    assert os.path.exists(out / "error:reS_ntop:-1" / "scores_th:2.000_min-visib:-1.000.json")
    cli("eval_pose_results_more.py", ",".join(six), "ev6", ["--score_only"])
    assert (out / "scores_bop19.json").read_bytes() == first
    # the BOP19 types: every file byte-identical to bop_eval.py's
    a, b = cli("bop_eval.py", "vsd,mssd,mspd,ad,add,adi", "ev_bop"), cli("eval_pose_results_more.py", "vsd,mssd,mspd,ad,add,adi",
                                                                          "ev_more")
    files = sorted(os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs)
    assert files == sorted(os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs)
    assert len(files) > 100
    _, mismatch, errs = filecmp.cmpfiles(str(a), str(b), files, shallow=False)
    assert not mismatch and not errs, mismatch[:5]
