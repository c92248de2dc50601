"""Generate tests/golden/ref_pose_error.npz by running the REFERENCE's own BOP pose-error functions (imported read-only
from the checkout that GDRN_REFERENCE_SRC names) on small seeded inputs:

  * misc.get_symmetry_transformations   (lib/pysixd/misc.py:234-282): no symmetry, discrete, continuous, both
  * pose_error.mssd / mspd / add / adi   (lib/pysixd/pose_error.py:131-179, 256-296)
  * pose_matching.match_poses_scene + score.calc_localization_scores on a seeded error set (score ties, several
    instances, missing estimates, inf errors, invalid GT), and misc.get_error_signature / get_score_signature
  * pose_error.vsd                       (lib/pysixd/pose_error.py:22-128) with renderer_type "python", fed by a stand-in
    renderer whose render_object returns stored depth maps: missing test depth, occlusion, an empty union, a pair with
    no overlap at all, and taus placed exactly on pixel distances, with and without normalisation by the diameter

Third-party imports the reference makes but which are absent here are stubbed exactly as in make_golden_ref_heads.py.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_pose_error.py
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_ref_heads as H  # noqa: E402

OUT = os.path.join(H.ROOT, "tests", "golden", "ref_pose_error.npz")

# models_info entries (BOP format, mm) for the symmetry cases
SYM_INFOS = {
    "none": {"diameter": 100.0},
    "discrete": {"diameter": 100.0, "symmetries_discrete": [
        [-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1],
        [1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 4.5, 0, 0, 0, 1]]},
    "continuous": {"diameter": 100.0, "symmetries_continuous": [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]},
    "both": {"diameter": 100.0, "symmetries_discrete": [[1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1]],
             "symmetries_continuous": [{"axis": [0.0, 0.6, 0.8], "offset": [1.5, -2.0, 3.0]}]},
}
MAX_SYM_DISC_STEP = 0.01
VSD_H, VSD_W = 24, 32


def rand_rot(rs):
    q = rs.randn(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


class StoredDepthRenderer:
    """renderer_type 'python' surface of pose_error.vsd: render_object(obj_id, R, t, fx, fy, cx, cy) -> {'depth'}.
    The depth of a pose is looked up by the pose's translation (each case uses distinct translations)."""

    def __init__(self):
        self.depths = {}

    def add(self, t, depth):
        self.depths[tuple(np.asarray(t, np.float64).ravel())] = depth

    def render_object(self, obj_id, R, t, fx, fy, cx, cy):
        return {"depth": self.depths[tuple(np.asarray(t, np.float64).ravel())]}


def vsd_cases(rs, misc):
    """Seeded depth triples (est, gt, test) [f32, mm] and the per-case (diameter, normalized) settings."""
    yy, xx = np.mgrid[0:VSD_H, 0:VSD_W]
    K = np.array([[40.0, 0, 15.3], [0, 41.0, 11.7], [0, 0, 1]])

    def blob(cx, cy, r, z0, slope):
        d = (z0 + slope * (xx - cx) + rs.rand(VSD_H, VSD_W) * 3).astype(np.float32)
        d[(xx - cx) ** 2 + (yy - cy) ** 2 > r * r] = 0
        return d

    cases = []
    # 0: plain overlap, scene = gt surface + noise with holes (missing test depth) and an occluder
    gt = blob(15, 12, 8, 700, 1.5)
    est = blob(17, 11, 8, 705, 1.4)
    test = np.where(gt > 0, gt + rs.randn(VSD_H, VSD_W).astype(np.float32) * 4, 900).astype(np.float32)
    test[3:8, 20:26] = 0                      # missing depth: counted as visible
    test[10:16, 4:10] = 500                   # occluder in front of both surfaces
    cases.append((est, gt, test))
    # 1: estimate far behind the scene surface (mostly invisible) and partly outside the gt silhouette
    gt = blob(10, 10, 7, 650, -1.0)
    est = blob(20, 13, 9, 800, 0.5)
    test = np.where(gt > 0, gt, 600).astype(np.float32)
    test[0:4, :] = 0
    cases.append((est, gt, test))
    # 2: empty union: both renders empty
    z = np.zeros((VSD_H, VSD_W), np.float32)
    cases.append((z.copy(), z.copy(), blob(15, 12, 8, 700, 0.0)))
    # 3: identical renders, scene with holes only -> every intersection distance is 0
    gt = blob(14, 12, 9, 720, 0.7)
    test = gt.copy()
    test[::3, ::4] = 0
    cases.append((gt.copy(), gt, test))
    # taus placed exactly on pixel distances of case 0 (step cost: dist >= tau counts)
    dist_gt = misc.depth_im_to_dist_im_fast(cases[0][1], K)
    dist_est = misc.depth_im_to_dist_im_fast(cases[0][0], K)
    both = (cases[0][0] > 0) & (cases[0][1] > 0)
    diffs = np.sort(np.abs(dist_gt[both] - dist_est[both]))
    return K, cases, diffs


def main():
    assert H.REF and os.path.isdir(H.REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    H.STUB_TOPLEVEL.update({"cv2", "numba", "six", "yaml", "png", "imageio"})
    sys.meta_path.insert(0, H.StubFinder())
    sys.path.insert(0, H.REF)
    for _n, _v in (("float", float), ("int", int), ("bool", bool)):
        if not hasattr(np, _n):
            setattr(np, _n, _v)
    from lib.pysixd import misc, pose_error, pose_matching, score

    rs = np.random.RandomState(2022)
    out = {}
    # --- symmetry transformations ---
    for name, info in SYM_INFOS.items():
        trans = misc.get_symmetry_transformations(info, MAX_SYM_DISC_STEP)
        out[f"sym_{name}"] = np.stack([np.hstack([np.asarray(s["R"], np.float64), np.asarray(s["t"], np.float64).reshape(3, 1)])
                                       for s in trans])
    # --- mssd / mspd / add / adi on seeded poses, points in mm ---
    pts = (rs.rand(300, 3) - 0.5) * np.array([80.0, 60.0, 40.0])
    K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])
    n_pairs = 6
    Re, te, Rg, tg = [], [], [], []
    for i in range(n_pairs):
        R_g = rand_rot(rs)
        t_g = np.array([rs.uniform(-80, 80), rs.uniform(-60, 60), rs.uniform(600, 1100)])
        dR = rand_rot(np.random.RandomState(100 + i)) if i == n_pairs - 1 else \
            np.linalg.qr(np.eye(3) + rs.randn(3, 3) * 0.05 * (i + 1))[0]
        dR = dR * np.sign(np.linalg.det(dR))
        Re.append(dR @ R_g)
        te.append(t_g + rs.randn(3) * 5 * (i + 1))
        Rg.append(R_g)
        tg.append(t_g)
    out["pe_pts"] = pts
    out["pe_K"] = K
    out["pe_R_est"], out["pe_t_est"] = np.stack(Re), np.stack(te)
    out["pe_R_gt"], out["pe_t_gt"] = np.stack(Rg), np.stack(tg)
    for name in SYM_INFOS:
        syms = misc.get_symmetry_transformations(SYM_INFOS[name], MAX_SYM_DISC_STEP)
        out[f"mssd_{name}"] = np.array([pose_error.mssd(Re[i], te[i].reshape(3, 1), Rg[i], tg[i].reshape(3, 1), pts, syms)
                                        for i in range(n_pairs)])
        out[f"mspd_{name}"] = np.array([pose_error.mspd(Re[i], te[i].reshape(3, 1), Rg[i], tg[i].reshape(3, 1), K, pts, syms)
                                        for i in range(n_pairs)])
    out["add"] = np.array([pose_error.add(Re[i], te[i].reshape(3, 1), Rg[i], tg[i].reshape(3, 1), pts) for i in range(n_pairs)])
    out["adi"] = np.array([pose_error.adi(Re[i], te[i].reshape(3, 1), Rg[i], tg[i].reshape(3, 1), pts) for i in range(n_pairs)])
    # --- vsd through the reference function with stored renders ---
    Kv, cases, diffs = vsd_cases(rs, misc)
    taus_exact = np.array([0.0, diffs[len(diffs) // 4], diffs[len(diffs) // 2], diffs[-1], diffs[-1] + 1.0])
    diameter = 87.5
    settings = [(taus_exact, False), (np.arange(0.05, 0.51, 0.05), True), (taus_exact / diameter, True)]
    errs = np.zeros((len(settings), len(cases), max(len(t) for t, _ in settings)))
    for si, (taus, normalized) in enumerate(settings):
        for ci, (est, gt, test) in enumerate(cases):
            ren = StoredDepthRenderer()
            t_e, t_g = np.array([1.0, 0, 500 + ci]), np.array([2.0, 0, 500 + ci])
            ren.add(t_e, est)
            ren.add(t_g, gt)
            e = pose_error.vsd(np.eye(3), t_e, np.eye(3), t_g, test, Kv, 15, list(taus), normalized, diameter, ren, 1,
                               "step", renderer_type="python")
            errs[si, ci, :len(taus)] = e
    out["vsd_K"] = Kv
    out["vsd_depth_est"] = np.stack([c[0] for c in cases])
    out["vsd_depth_gt"] = np.stack([c[1] for c in cases])
    out["vsd_depth_test"] = np.stack([c[2] for c in cases])
    out["vsd_taus_exact"] = taus_exact
    out["vsd_errors"] = errs
    out["vsd_delta"] = np.array(15.0)
    out["vsd_diameter"] = np.array(diameter)
    np.savez_compressed(OUT, **out)
    # --- match_poses_scene + calc_localization_scores on a seeded error set: score ties, several instances, missing
    # estimates, inf errors, invalid GT; and the error / score signatures ---
    srs = np.random.RandomState(7)
    scene_gt = {im: [{"obj_id": int(o)} for o in srs.choice([1, 2, 3], 4)] for im in range(5)}
    scene_gt_valid = {im: [bool(v) for v in srs.rand(4) > 0.2] for im in range(5)}
    scene_errs = []
    for im in range(5):
        for o in (1, 2, 3):
            gts = [g for g, gt in enumerate(scene_gt[im]) if gt["obj_id"] == o]
            for est_id in range(srs.randint(0, 4)):
                errs = {g: [float("inf") if srs.rand() < 0.15 else float(srs.rand() * 0.6)] for g in gts}
                scene_errs.append({"im_id": im, "obj_id": o, "est_id": est_id, "score": float(srs.choice([0.5, 0.7, 0.9])),
                                   "errors": errs})
    matching = []
    for th, n_top in (([0.3], -1), ([0.1], -1), ([0.3], 1)):
        m = pose_matching.match_poses_scene(3, scene_gt, scene_gt_valid, scene_errs, th, n_top)
        sc = score.calc_localization_scores([3, 4], [1, 2, 3], m, n_top, do_print=False)
        matching.append({"th": th, "n_top": n_top, "matches": m, "scores": sc})
    signatures = {"error": [misc.get_error_signature("vsd", -1, vsd_delta=15, vsd_tau=t) for t in np.arange(0.05, 0.51, 0.05)]
                   + [misc.get_error_signature("vsd", 1, vsd_delta=5, vsd_tau=float("inf")),
                      misc.get_error_signature("mssd", -1), misc.get_error_signature("ad", 0)],
                  "score": [misc.get_score_signature([th], -1) for th in np.arange(5, 51, 5)]
                   + [misc.get_score_signature([0.02], 0.1), misc.get_score_signature([2, 5], -1)]}
    meta_extra = {"scene_gt": {str(k): v for k, v in scene_gt.items()},
                  "scene_gt_valid": {str(k): v for k, v in scene_gt_valid.items()},
                  "scene_errs": scene_errs, "matching": matching, "signatures": signatures}
    meta = {**meta_extra, "max_sym_disc_step": MAX_SYM_DISC_STEP, "sym_infos": SYM_INFOS,
            "vsd_settings": [{"taus": "exact" if t is taus_exact else ("exact/diameter" if si == 2 else "bop19"),
                              "normalized_by_diameter": n} for si, (t, n) in enumerate(settings)]}
    with open(OUT[:-4] + ".json", "w") as f:
        json.dump(meta, f, indent=None, default=lambda x: {str(k): v for k, v in x.items()} if isinstance(x, dict) else x)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
