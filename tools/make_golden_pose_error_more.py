"""Generate tests/golden/ref_pose_error_more.npz (+ .json) by running the REFERENCE's own pose-error functions of
eval_pose_results_more.py (imported read-only from the checkout that GDRN_REFERENCE_SRC names) on small seeded inputs:

  * pose_error.re / re_sym / te / te_sym / arp_2d / arp_2d_sym / add / adi (lib/pysixd/pose_error.py:183-445) over the
    four symmetry cases of make_golden_pose_error.py, on seeded random poses, an exact-identity pair (the trace clamp),
    a 180 degree pair, a 1e-4 rad pair, an estimate 1 m off and a pose with some model points behind the camera
  * misc.get_symmetry_transformations for those cases (the continuous sets hold no identity)
  * the error table (p["errors"]) and default --error_types of scripts/eval_pose_results_more.py and the normalisation
    lists of scripts/eval_calc_scores.py.  Those scripts parse arguments and evaluate at import, so the values are
    taken from their syntax trees and evaluated with numpy only.

Third-party imports the reference makes but which are absent here are stubbed as in make_golden_pose_error.py.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_pose_error_more.py
"""
import ast
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_pose_error as G  # noqa: E402
import make_golden_ref_heads as H  # noqa: E402

OUT = os.path.join(H.ROOT, "tests", "golden", "ref_pose_error_more.npz")
SCRIPTS = os.path.join("lib", "pysixd", "scripts")


def _p_dict(tree):
    """The value node of the module-level `p = {...}` assignment."""
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "p" for t in node.targets):
            return node.value
    raise KeyError("p")


def _dict_item(dict_node, key):
    for k, v in zip(dict_node.keys, dict_node.values):
        if isinstance(k, ast.Constant) and k.value == key:
            return v
    raise KeyError(key)


def _eval(node):
    return eval(compile(ast.Expression(node), "<ref>", "eval"), {"np": np})


def reference_tables():
    with open(os.path.join(H.REF, SCRIPTS, "eval_pose_results_more.py")) as f:
        more = ast.parse(f.read())
    errors = _eval(_dict_item(_p_dict(more), "errors"))
    default_types = None
    for node in ast.walk(more):
        if (isinstance(node, ast.Call) and getattr(node.func, "attr", "") == "add_argument" and node.args
                and isinstance(node.args[0], ast.Constant) and node.args[0].value == "--error_types"):
            default_types = _eval(next(k.value for k in node.keywords if k.arg == "default"))
    with open(os.path.join(H.REF, SCRIPTS, "eval_calc_scores.py")) as f:
        scores_p = _p_dict(ast.parse(f.read()))
    return {"errors": [{"type": e["type"], "n_top": e["n_top"],
                        "correct_th": [[float(t) for t in th] for th in e["correct_th"]]} for e in errors],
            "default_error_types": default_types,
            "normalized_by_diameter": _eval(_dict_item(scores_p, "normalized_by_diameter")),
            "normalized_by_im_width": _eval(_dict_item(scores_p, "normalized_by_im_width"))}


def axis_rot(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * Kx + (1 - np.cos(angle)) * Kx @ Kx


def pose_cases(rs):
    """-> names, R_est, t_est, R_gt, t_gt (t in mm)."""
    names, Re, te, Rg, tg = [], [], [], [], []

    def add(name, R_e, t_e, R_g, t_g):
        names.append(name)
        Re.append(R_e)
        te.append(np.asarray(t_e, np.float64))
        Rg.append(R_g)
        tg.append(np.asarray(t_g, np.float64))

    for i in range(4):
        R_g = G.rand_rot(rs)
        t_g = np.array([rs.uniform(-80, 80), rs.uniform(-60, 60), rs.uniform(600, 1100)])
        dR = np.linalg.qr(np.eye(3) + rs.randn(3, 3) * 0.1 * (i + 1))[0]
        dR = dR * np.sign(np.linalg.det(dR))
        add("random%d" % i, dR @ R_g, t_g + rs.randn(3) * 8 * (i + 1), R_g, t_g)
    R_g = G.rand_rot(rs)
    t_g = np.array([20.0, -15.0, 800.0])
    add("identity", R_g.copy(), t_g.copy(), R_g, t_g)
    add("rot180", axis_rot([0.3, -0.5, 0.8], np.pi) @ R_g, t_g + [1.0, 2.0, 3.0], R_g, t_g)
    add("small_angle", axis_rot([0.6, 0.0, 0.8], 1e-4) @ R_g, t_g + [0.01, 0.0, 0.02], R_g, t_g)
    add("off_1m", G.rand_rot(rs) @ R_g, t_g + [0.0, 0.0, 1000.0], R_g, t_g)
    R_g = G.rand_rot(rs)
    add("behind_camera", axis_rot([1.0, 0.0, 0.0], 0.2) @ R_g, [5.0, -4.0, 12.0], R_g, [-3.0, 2.0, 10.0])
    return names, np.stack(Re), np.stack(te), np.stack(Rg), np.stack(tg)


def main():
    assert H.REF and os.path.isdir(H.REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    H.STUB_TOPLEVEL.update({"cv2", "numba", "six", "yaml", "png", "imageio"})
    sys.meta_path.insert(0, H.StubFinder())
    sys.path.insert(0, H.REF)
    for _n, _v in (("float", float), ("int", int), ("bool", bool)):
        if not hasattr(np, _n):
            setattr(np, _n, _v)
    from lib.pysixd import misc, pose_error

    rs = np.random.RandomState(2023)
    out = {}
    pts = (rs.rand(200, 3) - 0.5) * np.array([80.0, 60.0, 40.0])
    K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])
    names, Re, te, Rg, tg = pose_cases(rs)
    P = len(names)
    for R, t in ((Re[-1], te[-1]), (Rg[-1], tg[-1])):
        cam_z = (pts @ R.T + t)[:, 2]
        assert (cam_z < 0).any() and (cam_z > 0).any(), "the last case needs points on both sides of the camera"
    a = [(Re[i], te[i].reshape(3, 1), Rg[i], tg[i].reshape(3, 1)) for i in range(P)]
    out["pts"], out["K"] = pts, K
    out["R_est"], out["t_est"], out["R_gt"], out["t_gt"] = Re, te, Rg, tg
    out["re"] = np.array([pose_error.re(x[0], x[2]) for x in a])
    out["te"] = np.array([pose_error.te(x[1], x[3]) for x in a])
    out["arp_2d"] = np.array([pose_error.arp_2d(*x, pts, K) for x in a])
    out["add"] = np.array([pose_error.add(*x, pts) for x in a])
    out["adi"] = np.array([pose_error.adi(*x, pts) for x in a])
    for name, info in G.SYM_INFOS.items():
        syms = misc.get_symmetry_transformations(info, G.MAX_SYM_DISC_STEP)
        out[f"sym_{name}"] = np.stack([np.hstack([np.asarray(s["R"], np.float64), np.asarray(s["t"], np.float64).reshape(3, 1)])
                                       for s in syms])
        out[f"re_sym_{name}"] = np.array([pose_error.re_sym(x[0], x[2], syms) for x in a])
        out[f"te_sym_{name}"] = np.array([pose_error.te_sym(x[1], x[3], x[2], syms) for x in a])
        out[f"arp_2d_sym_{name}"] = np.array([pose_error.arp_2d_sym(*x, pts, K, syms) for x in a])
    np.savez_compressed(OUT, **out)
    meta = {"cases": names, "max_sym_disc_step": G.MAX_SYM_DISC_STEP, "sym_infos": G.SYM_INFOS, **reference_tables()}
    with open(OUT[:-4] + ".json", "w") as f:
        json.dump(meta, f, indent=None)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
