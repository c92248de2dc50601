"""GT and estimated pose outlines (gdrnpp_bop2022_b200.vis_poses_full, EGLRenderer.render(background=)): the host
pieces against the reference's own get_edge, mask2bbox_xyxy and vis_image_bboxes_cv2 (tests/golden/ref_vis_poses_full.npz,
tools/make_golden_vis_poses_full.py) and against restatements of the scripts' arithmetic; the kernels against cv2 and
the NumPy restatement; the CLI end to end against a host driver that follows the scripts' loop literally."""
import json
import os

import numpy as np
import pytest

from conftest import ROOT
from gdrnpp_bop2022_b200 import gt_info
from gdrnpp_bop2022_b200 import vis_poses_full as VF
from gdrnpp_bop2022_b200._lib import GdrnError
from oracle import vis_poses_full_oracle as O

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_vis_poses_full.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def test_host_get_edge_and_box_match_reference_fixture(golden):
    g = golden
    for bw in (1, 3):
        for m, e in zip(g["masks"], g[f"edges_bw{bw}"]):
            assert np.array_equal(O.get_edge(m, bw), e), bw
    for m, b in zip(g["masks"], g["bbox_xyxy"]):
        if m.any():
            assert O.mask2bbox_xyxy(m) == list(b)
    # the fixture covers what it claims: every border touched, an empty and a full mask
    ms = g["masks"].astype(bool)
    assert ms[:, 0].any() and ms[:, -1].any() and ms[:, :, 0].any() and ms[:, :, -1].any()
    assert not ms[-1].any() and ms[-2].all() and not g["edges_bw3"][-2].any()


def test_box_drawing_matches_reference_fixture(golden):
    g = golden
    out = VF.draw_bboxes(g["image"], list(g["boxes"]), [str(s) for s in g["labels"]])
    assert np.array_equal(out, g["boxed"])
    assert not np.array_equal(out, g["image"])
    boxes, labels = VF.det_boxes([{"bbox_est": [1.5, 2.0, 10.0, 4.25], "obj_id": 7, "score": 0.3},
                                  {"bbox_est": [0, 0, 1, 1], "obj_id": 2, "score": 0.29}])
    assert labels == ["7"] and np.array_equal(boxes[0], [1.5, 2.0, 11.5, 6.25])


def _zoom_restated(minx, miny, maxx, maxy, K, imH, imW, out_size):
    """ycbv_2_vis_poses.py:174-190 and get_affine_transform (core/utils/data_utils.py:136-184) with cv2's solver."""
    import cv2

    center = np.array([(minx + maxx) / 2, (miny + maxy) / 2])
    scale = max(maxx - minx, maxy - miny) * 1.5
    cminx, cminy = max(0, center[0] - scale / 2), max(0, center[1] - scale / 2)
    cmaxx, cmaxy = min(imW - 1, center[0] + scale / 2), min(imH - 1, center[1] + scale / 2)
    scale = min(scale, min(cmaxx - cminx, cmaxy - cminy))
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0] = center
    src[1] = center + np.array([0.0, scale * -0.5])
    dst[0] = [out_size * 0.5, out_size * 0.5]
    dst[1] = np.array([out_size * 0.5, out_size * 0.5], np.float32) + np.array([0, out_size * -0.5], np.float32)
    for p in (src, dst):
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], np.float32)
    M = cv2.getAffineTransform(src, dst)
    Kz = np.asarray(K, np.float32).copy()
    Kz[0, 2] = np.float32(np.float64(Kz[0, 2]) - (center[0] - scale / 2))
    Kz[1, 2] = np.float32(np.float64(Kz[1, 2]) - (center[1] - scale / 2))
    # the in-place row update: when the clip picked an integer extent, scale is a Python int and out_size / scale a
    # Python float, which NumPy multiplies in f32; otherwise scale is np.float64 and the product is formed in f64
    for r in (0, 1):
        if isinstance(scale, int):
            Kz[r] = Kz[r] * np.float32(out_size / scale)
        else:
            Kz[r] = (Kz[r].astype(np.float64) * (out_size / scale)).astype(np.float32)
    return center, scale, M, Kz


def test_zoom_arithmetic_matches_restatement():
    rs = np.random.RandomState(3)
    K = np.array([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]], np.float32)
    cases = [(0, 0, 639, 479), (300, 200, 301, 201), (5, 400, 80, 479), (600, 10, 639, 30), (100, 100, 101, 100)]
    cases += [tuple(sorted(rs.randint(0, 640, 2))[i // 2] if i % 2 == 0 else sorted(rs.randint(0, 480, 2))[i // 2]
                    for i in range(4)) for _ in range(20)]
    kinds = set()
    for box in cases:
        minx, miny, maxx, maxy = box
        c, s, M, Kz = VF.zoom_params(box, K, 480, 640, 512)
        c2, s2, M2, Kz2 = _zoom_restated(np.int64(minx), np.int64(miny), np.int64(maxx), np.int64(maxy), K, 480, 640,
                                         512)
        assert np.array_equal(c, c2) and s == s2, box
        np.testing.assert_allclose(M, M2, rtol=0, atol=1e-9)
        assert np.array_equal(Kz, Kz2) and Kz.dtype == np.float32, box
        kinds.add(type(s2).__name__)
    assert kinds == {"int", "float64"}
    with pytest.raises(GdrnError, match="zoom box .* one pixel"):
        VF.zoom_params((7, 9, 7, 9), K, 480, 640)


def _split(root, **kw):
    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    kw.setdefault("H", 48)
    kw.setdefault("W", 64)
    write_bop_tree(root, dataset="ycbv", num_images=5, num_scenes=2, dets_per_image=4, obj_ids=[1, 2, 3, 4], **kw)
    return gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "ycbv", "test")


def _write_csv(path, rows, header="scene_id,im_id,obj_id,score,R,t,time"):
    with open(path, "w") as f:
        f.write(header + "\n")
        for scene_id, im_id, obj_id, score, R, t in rows:
            f.write("{},{},{},{},{},{},0.1\n".format(scene_id, im_id, obj_id, score,
                                                      " ".join("%.9g" % v for v in np.ravel(R)),
                                                      " ".join("%.9g" % v for v in np.ravel(t))))


def test_csv_filtering_and_image_selection(tmp_path):
    sp = _split(str(tmp_path / "d"))
    ims = VF.plan(sp)   # no results: every registrar image, GT only
    assert [(s, i) for s, i, *_ in ims] == [(1, 1), (1, 4), (1, 7), (2, 1), (2, 4)]
    R = np.eye(3)
    csv = str(tmp_path / "r.csv")
    _write_csv(csv, [(1, 1, 1, 0.3, R, [10.0, -20.0, 800.0]), (1, 1, 2, 0.2999, R, [0, 0, 900]),
                     (1, 4, 3, 0.1, R, [0, 0, 700]), (2, 4, 2, 0.95, R, [1, 2, 3])])
    res = VF.load_results(csv)
    assert sorted(res) == [(1, 1), (1, 4), (2, 4)]
    np.testing.assert_array_equal(res[(1, 1)][0]["t"], np.array([10.0, -20.0, 800.0]) / 1000)
    assert [r["obj_id"] for r in VF.kept_estimates(res[(1, 1)])] == [1]
    ims = VF.plan(sp, results=res)
    # images without rows are skipped; (1, 4) stays with no estimate drawn (its only row is below the threshold)
    assert [(s, i) for s, i, *_ in ims] == [(1, 1), (1, 4), (2, 4)]
    est = {(s, i): [p for p in insts if not p["gt"]] for s, i, _, _, _, _, insts, _ in ims}
    assert [p["obj_id"] for p in est[(1, 1)]] == [1] and est[(1, 4)] == []
    assert [p["obj_id"] for p in VF.plan(sp, results=res, score_thr=0.1)[1][6] if not p["gt"]] == [3]
    # the registrar's GT rule: an empty mask_visib drops the instance, an image without instances is dropped
    path = os.path.join(sp["split_path"], "000001", "scene_gt_info.json")
    with open(path) as f:
        info = json.load(f)
    for g in info["1"]:
        g["px_count_visib"] = 0
    info["4"][1]["px_count_visib"] = 0
    with open(path, "w") as f:
        json.dump(info, f)
    ims = {(s, i): insts for s, i, _, _, _, _, insts, _ in VF.plan(sp, results=res)}
    assert (1, 1) not in ims and len([p for p in ims[(1, 4)] if p["gt"]]) == 3
    gt = [p for p in ims[(2, 4)] if p["gt"]]
    assert gt[0]["R"].dtype == np.float32 and gt[0]["t"].dtype == np.float32


def test_cli_parsing_and_rejections(tmp_path):
    a = VF.parse_args(["--dataset", "tudl", "--result_filename", "x.csv", "--det_file", "d.json", "--score_thr", "0.5",
                       "--scene_ids", "1,2", "--max_bytes", "1000"])
    assert (a.dataset, a.det_file, a.score_thr, a.scene_ids, a.max_bytes, a.zoom, a.out_size) == \
        ("tudl", "d.json", 0.5, [1, 2], 1000, False, 512)
    for bad in (["--dataset", "ycbv"], ["--result_filename", "x.csv"], ["--dataset", "nope", "--result_filename", "x"],
                ["--dataset", "ycbv", "--result_filename", "x", "--zoom", "--det_file", "d.json"],
                ["--dataset", "ycbv", "--result_filename", "x", "--out_size", "0"]):
        with pytest.raises(SystemExit):
            VF.parse_args(bad)
    csv = str(tmp_path / "bad.csv")
    _write_csv(csv, [(1, 1, 1, 0.9, np.eye(3), [0, 0, 1])], header="scene_id,im_id,obj_id,score,R,t")
    with pytest.raises(GdrnError, match="missing column.*time"):
        VF.load_results(csv)
    sp = _split(str(tmp_path / "a"))
    models = os.path.join(sp["base_path"], "models_eval")
    res = {(1, 1): [{"obj_id": 9, "score": 0.9, "R": np.eye(3), "t": np.array([0, 0, 1.0])}]}
    with pytest.raises(GdrnError, match="obj_id 9: no model file"):
        VF.run_split(sp, models, str(tmp_path / "o"), res, device="cpu")
    os.remove(os.path.join(sp["split_path"], "000001", "rgb", "000004.png"))
    with pytest.raises(GdrnError, match="missing rgb image .*000004.png"):
        VF.run_split(sp, models, str(tmp_path / "o"), {(1, 4): res[(1, 1)]}, device="cpu")
    with pytest.raises(GdrnError, match="--det_file with --zoom"):
        VF.run_split(sp, models, str(tmp_path / "o"), res, zoom=True, dets={}, device="cpu")
    for s in ("000001", "000002"):   # a split without GT (as ITODD test): estimates only, and no zoom
        os.remove(os.path.join(sp["split_path"], s, "scene_gt.json"))
    ims = VF.plan(sp, results={(2, 4): res[(1, 1)]})
    assert [(i[0], i[1], len(i[6]), i[7]) for i in ims] == [(2, 4, 1, None)]
    with pytest.raises(GdrnError, match="--zoom: split .* has no GT"):
        VF.plan(sp, results=res, zoom=True)


def test_non_uint8_background_still_raises():
    import torch

    from gdrnpp_bop2022_b200.renderer import EGLRenderer

    egl = EGLRenderer([], K=np.eye(3), width=4, height=4, device="cpu")
    for bg in (np.zeros((4, 4, 3), np.float32), np.zeros((4, 4), np.int16), torch.zeros((4, 4, 3))):
        with pytest.raises(NotImplementedError, match="background"):
            egl.render([0], [np.eye(4)[:3]], background=bg)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _egl(dev, H, W, textured=False):
    """An EGLRenderer over two meshes (metres): a box and a vertex-coloured icosahedron."""
    from gdrnpp_bop2022_b200.renderer import EGLRenderer, Model3D, calc_normals
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    box = np.array([[x, y, z] for x in (-0.03, 0.03) for y in (-0.02, 0.02) for z in (-0.025, 0.025)], np.float32)
    bf = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                   [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    v, f = make_icosphere_mesh(2, (0.05, 0.04, 0.06))
    v = np.asarray(v, np.float32)
    cols = np.random.RandomState(1).rand(len(v), 3).astype(np.float32)
    ms = [Model3D(box, bf, device=dev, normals=calc_normals(box)),
          Model3D(v, f, device=dev, colors=cols, normals=calc_normals(v))]
    return EGLRenderer(ms, K=np.eye(3), width=W, height=H, device=dev)


def _pose(rs, z):
    import cv2

    R = cv2.Rodrigues(rs.uniform(-1, 1, 3))[0]
    return np.hstack([R, np.array([[rs.uniform(-0.05, 0.05)], [rs.uniform(-0.04, 0.04)], [z]])]).astype(np.float32)


@pytest.mark.gpu
def test_background_fills_uncovered_pixels_only(lib, dev):
    import torch

    H, W = 61, 83
    egl = _egl(dev, H, W)
    rs = np.random.RandomState(11)
    K = np.array([[90.0, 0, 40.3], [0, 92.0, 29.7], [0, 0, 1]], np.float32)
    poses = [_pose(rs, 0.5), _pose(rs, 0.45)]
    bg3 = rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
    bg2 = rs.randint(0, 256, (H, W)).astype(np.uint8)
    t = lambda: torch.full((H, W, 4), -7.0, device=dev)   # noqa: E731
    for to_bgr in (True, False):
        for to_255 in (True, False):
            for bg in (bg3, bg2, torch.from_numpy(bg3).to(dev)):
                ref = {k: t() for k in ("image", "seg", "pc_obj", "pc_cam", "normal")}
                got = {k: t() for k in ref}
                d0 = egl.render([0, 1], poses, K=K, to_bgr=to_bgr, to_255=to_255, **{k + "_tensor": v for k, v in ref.items()})
                d1 = egl.render([0, 1], poses, K=K, to_bgr=to_bgr, to_255=to_255, background=bg,
                                **{k + "_tensor": v for k, v in got.items()})
                assert torch.equal(d0, d1)
                for k in ("seg", "pc_obj", "pc_cam", "normal"):
                    assert torch.equal(ref[k], got[k]), k
                cov = (d0 > 0).cpu().numpy()
                assert cov.any() and (~cov).any()
                a, b = ref["image"].cpu().numpy(), got["image"].cpu().numpy()
                assert np.array_equal(a[cov], b[cov])
                v = np.asarray(bg.cpu() if torch.is_tensor(bg) else bg)
                v = np.repeat(v[..., None], 3, axis=2) if v.ndim == 2 else v
                e = v.astype(np.float32) / np.float32(255)
                if to_bgr:
                    e = e[..., ::-1]
                e = np.concatenate([e, np.ones((H, W, 1), np.float32)], axis=2)
                if to_255:
                    e = e * np.float32(255)
                assert np.array_equal(b[~cov], e[~cov])
    # no instance: the background alone; another size is refused
    img = t()
    egl.render([], [], K=K, image_tensor=img, background=bg3)
    assert np.array_equal(img[..., :3].cpu().numpy(), (bg3.astype(np.float32) / np.float32(255))[..., ::-1] * np.float32(255))
    with pytest.raises(ValueError, match="background"):
        egl.render([0], poses[:1], K=K, image_tensor=t(), background=bg3[:-1])


@pytest.mark.gpu
def test_gray3_matches_cv2(lib, dev):
    import cv2
    import torch

    rs = np.random.RandomState(4)
    for N, H, W in ((1, 1, 1), (3, 7, 13), (2, 129, 77)):
        bgr = rs.randint(0, 256, (N, H, W, 3)).astype(np.uint8)
        exp = np.stack([np.repeat(cv2.cvtColor(im, cv2.COLOR_BGR2GRAY)[..., None], 3, axis=2) for im in bgr])
        assert np.array_equal(exp, O.bgr2gray3(bgr))
        got = VF.gray3(torch.from_numpy(bgr).to(dev), rgb_order=False).cpu().numpy()
        assert np.array_equal(got, exp)
        got = VF.gray3(torch.from_numpy(np.ascontiguousarray(bgr[..., ::-1])).to(dev), rgb_order=True).cpu().numpy()
        assert np.array_equal(got, exp)


@pytest.mark.gpu
def test_silhouettes_equal_single_instance_seg(lib, dev):
    import torch

    from gdrnpp_bop2022_b200.renderer import render_meshes

    H, W = 57, 71
    egl = _egl(dev, H, W)
    rs = np.random.RandomState(8)
    K = np.array([[80.0, 0, 33.1], [0, 81.0, 30.2], [0, 0, 1]], np.float32)
    objs = [0, 1, 1, 0, 1]
    poses = [_pose(rs, z) for z in (0.5, 0.3, 0.26, 0.9, 0.4)]
    poses[3][0, 3] = 0.3    # partly off the image
    ids = torch.tensor([egl.models[o].mesh_id for o in objs], dtype=torch.int32, device=dev)
    cov = render_meshes(ids, torch.from_numpy(np.stack(poses)).to(dev), torch.from_numpy(np.stack([K] * 5)).to(dev), H, W,
                        VF.ZNEAR, VF.ZFAR)
    seg = torch.zeros((H, W, 4), device=dev)
    for k, (o, p) in enumerate(zip(objs, poses)):
        egl.render([o], [p], K=K, seg_tensor=seg)
        m = (seg[..., 0] > 0).cpu().numpy()
        assert np.array_equal(m, (cov[k] != 0).cpu().numpy()), k
        assert m.any()


@pytest.mark.gpu
def test_outlines_kernel_matches_restatement(lib, dev, golden):
    import torch

    ms = golden["masks"]
    H, W = ms.shape[1:]
    rs = np.random.RandomState(6)
    # per image: (GT mask indices, estimate mask indices); overlapping, border-touching, full, empty, no GT, no estimate
    scenes = [([0, 4, 5], [1, 6, 0]), ([], [2, 7, 10]), ([3, 8, 9], []), ([], []), ([11, 10], [11])]
    covers, is_gt, off = [], [], [0]
    for g, e in scenes:
        covers += [ms[k] for k in g] + [ms[k] for k in e]
        is_gt += [1] * len(g) + [0] * len(e)
        off.append(off[-1] + len(g) + len(e))
    shaded = rs.rand(len(scenes), H, W, 3).astype(np.float32)
    shaded[0, :5] = (np.arange(5 * W * 3).reshape(5, W, 3) % 256).astype(np.float32) / np.float32(255)   # exact v/255
    shaded[1, :3] = np.float32(0.5) / np.float32(255) * np.arange(3 * W * 3).reshape(3, W, 3) % 1   # ties at .5
    cov = torch.from_numpy(np.stack(covers).astype(np.float32) * rs.uniform(0.3, 2.0)).to(dev)
    out = VF.outlines(torch.from_numpy(shaded).to(dev), cov, torch.tensor(off, dtype=torch.int32, device=dev),
                      torch.tensor(is_gt, dtype=torch.uint8, device=dev)).cpu().numpy()
    for j, (g, e) in enumerate(scenes):
        exp = O.composite(shaded[j], [ms[k] for k in g], [ms[k] for k in e])
        assert np.array_equal(out[j], exp), j
    assert (out == (0, 255, 0)).all(-1).any() and (out == (255, 0, 0)).all(-1).any()
    empty = VF.outlines(torch.from_numpy(shaded[:2]).to(dev), None, torch.zeros(3, dtype=torch.int32, device=dev),
                        None).cpu().numpy()
    assert np.array_equal(empty, np.stack([O.ren_bgr(s) for s in shaded[:2]]))


# ---- the CLI end to end ---------------------------------------------------------------------------------------------
def _annotated_split(root, dev, H=48, W=64):
    """The synthetic split with scene_gt_info.json and mask_visib/ written by gt_info from renders of its models."""
    sp = _split(root, H=H, W=W)
    gt_info.run_split(sp, os.path.join(sp["base_path"], "models_eval"), device=dev)
    return sp


def _results(sp, path, rs):
    """Estimates: each kept GT instance moved and turned (score >= 0.3), plus low-score rows; image (1, 7) has only
    low-score rows, (2, 1) has none."""
    import cv2

    rows = []
    for scene_id, ims in gt_info.plan_split(sp):
        for im in ims:
            if (scene_id, im["im_id"]) == (2, 1):
                continue
            for k, g in enumerate(im["gts"]):
                dR = cv2.Rodrigues(rs.uniform(-0.3, 0.3, 3))[0]
                t = np.asarray(g["cam_t_m2c"], np.float64).ravel() + rs.uniform(-20, 20, 3)
                low = (scene_id, im["im_id"]) == (1, 7) or k == 1
                rows.append((scene_id, im["im_id"], g["obj_id"], 0.2 if low else 0.3 + 0.1 * k,
                             dR @ np.asarray(g["cam_R_m2c"]).reshape(3, 3), t))
    _write_csv(path, rows)


def _host_driver(sp, csv, zoom, dets, out_size=64):
    """The scripts' loop literally: EGLRenderer renders the estimates over the grey image, then each instance alone
    (seg_tensor > 0), NumPy get_edge paints its edges, cv2 draws the boxes.  -> {stem: (vis0, vis1)} BGR."""
    import cv2
    import torch

    from gdrnpp_bop2022_b200 import bop_eval
    from gdrnpp_bop2022_b200.renderer import EGLRenderer

    models = os.path.join(sp["base_path"], "models_eval")
    ids = [1, 2, 3, 4]
    ren = None
    preds = VF.load_results(csv)
    targets = sorted({(t["scene_id"], t["im_id"]) for t in bop_eval.load_json(os.path.join(sp["base_path"],
                                                                                             "test_targets_bop19.json"))})
    out = {}
    for scene_id, im_id in targets:
        sdir = os.path.join(sp["split_path"], "{:06d}".format(scene_id))
        gts = bop_eval.load_json(os.path.join(sdir, "scene_gt.json"))[str(im_id)]
        infos = bop_eval.load_json(os.path.join(sdir, "scene_gt_info.json"))[str(im_id)]
        K = np.array(bop_eval.load_json(os.path.join(sdir, "scene_camera.json"))[str(im_id)]["cam_K"],
                     np.float32).reshape(3, 3)
        annos = []
        for k, (g, inf) in enumerate(zip(gts, infos)):
            m = cv2.imread(os.path.join(sdir, "mask_visib", "{:06d}_{:06d}.png".format(im_id, k)), cv2.IMREAD_UNCHANGED)
            assert (m.sum() >= 3) == (inf["px_count_visib"] > 0)
            if m.sum() < 3:
                continue
            annos.append((g, m))
        if not annos or (scene_id, im_id) not in preds:
            continue
        img = cv2.imread(os.path.join(sdir, "rgb", "{:06d}.png".format(im_id)))
        imH, imW = img.shape[:2]
        if zoom:
            fg = sum(m for _, m in annos).astype(bool).astype(np.uint8)
            box = O.mask2bbox_xyxy(fg)
            _, _, M, K = VF.zoom_params(box, K, imH, imW, out_size)
            img = cv2.warpAffine(img, M, (out_size, out_size), flags=cv2.INTER_LINEAR)
        H, W = img.shape[:2]
        if ren is None or (ren.height, ren.width) != (H, W):
            ren = EGLRenderer([os.path.join(models, "obj_{:06d}.ply".format(o)) for o in ids], model_ids=ids,
                              vertex_scale=0.001, width=W, height=H)
        image_tensor = torch.empty((H, W, 4), device="cuda")
        seg_tensor = torch.empty((H, W, 4), device="cuda")
        est = [(p["obj_id"], np.hstack([p["R"], p["t"].reshape(3, 1)])) for p in preds[(scene_id, im_id)]
               if p["score"] >= 0.3]
        gray = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)[..., None]
        ren.render([o for o, _ in est], [p for _, p in est], K=K, image_tensor=image_tensor,
                   background=np.concatenate([gray, gray, gray], axis=2))
        ren_bgr = (image_tensor[:, :, :3].cpu().numpy() + 0.5).astype("uint8")
        gt_poses = [(g["obj_id"], np.hstack([np.array(g["cam_R_m2c"], np.float32).reshape(3, 3),
                                             (np.array(g["cam_t_m2c"], np.float32) / 1000.0).reshape(3, 1)]))
                    for g, _ in annos]
        for lst, col in ((gt_poses, (255, 0, 0)), (est, (0, 255, 0))):
            for o, p in lst:
                ren.render([o], [p], K=K, seg_tensor=seg_tensor)
                ren_bgr[O.get_edge((seg_tensor[:, :, 0].cpu().numpy() > 0).astype("uint8"), 3)] = col
        vis0 = img
        if dets is not None:
            vis0 = VF.draw_bboxes(img, *VF.det_boxes(dets["{}/{}".format(scene_id, im_id)]))
        out["{}_{:06d}".format(scene_id, im_id)] = (vis0, ren_bgr)
    return out


def _read_pngs(d):
    import cv2

    return {f[:-4]: cv2.imread(os.path.join(d, f), cv2.IMREAD_UNCHANGED) for f in sorted(os.listdir(d))
            if f.endswith(".png")}


@pytest.mark.gpu
def test_cli_end_to_end_matches_the_scripts_loop(lib, dev, tmp_path):
    root = str(tmp_path / "datasets")
    sp = _annotated_split(root, dev)
    # the zoom box assumption: union of the kept bbox_visib == mask2bbox_xyxy of the union of the mask_visib PNGs
    import cv2

    for (scene_id, im_id, *_r, box) in VF.plan(sp):
        sdir = os.path.join(sp["split_path"], "{:06d}".format(scene_id))
        n = len(json.load(open(os.path.join(sdir, "scene_gt.json")))[str(im_id)])
        fg = sum(cv2.imread(os.path.join(sdir, "mask_visib", "{:06d}_{:06d}.png".format(im_id, k)), cv2.IMREAD_UNCHANGED)
                 .astype(np.int64) for k in range(n)) > 0
        assert tuple(O.mask2bbox_xyxy(fg)) == box
    csv = str(tmp_path / "gdrn_ycbv-test.csv")
    _results(sp, csv, np.random.RandomState(5))
    det_file = os.path.join(sp["split_path"], "test_bboxes", "dets.json")
    dets = json.load(open(det_file))
    base = ["--dataset", "ycbv", "--result_filename", csv, "--datasets_path", os.path.join(root, "BOP_DATASETS"),
            "--models_dir", os.path.join(sp["base_path"], "models_eval")]
    for name, extra, zoom, d in (("full", [], False, None), ("zoom", ["--zoom", "--out_size", "64"], True, None),
                                 ("det", ["--det_file", det_file], False, dets)):
        vis = str(tmp_path / name)
        r = VF.main(base + ["--vis_path", vis] + extra)
        got = _read_pngs(os.path.join(vis, "gdrn_ycbv-test"))
        exp = _host_driver(sp, csv, zoom, d)
        assert r["images"] == len(exp) == 4 and "2_000001" not in exp and "1_000007" in exp
        assert sorted(got) == sorted(k + s for k in exp for s in ("_vis0", "_vis1")), name
        for k, (v0, v1) in exp.items():
            assert np.array_equal(got[k + "_vis0"], v0), (name, k)
            assert np.array_equal(got[k + "_vis1"], v1), (name, k)
            assert (v1 == (0, 255, 0)).all(-1).any() or k == "1_000007"
            assert (v1 == (255, 0, 0)).all(-1).any()


@pytest.mark.gpu
def test_batches_write_identical_files(lib, dev, tmp_path):
    root = str(tmp_path / "datasets")
    sp = _annotated_split(root, dev)
    csv = str(tmp_path / "r.csv")
    _results(sp, csv, np.random.RandomState(9))
    res = VF.load_results(csv)
    models = os.path.join(sp["base_path"], "models_eval")
    for zoom in (False, True):
        outs = []
        for mb in (1, 1 << 30):
            d = str(tmp_path / "o{}_{}".format(int(zoom), mb))
            VF.run_split(sp, models, d, res, zoom=zoom, out_size=40, max_bytes=mb, device=dev)
            outs.append(_read_pngs(d))
        assert sorted(outs[0]) == sorted(outs[1]) and len(outs[0]) == 8
        for k in outs[0]:
            assert np.array_equal(outs[0][k], outs[1][k]), (zoom, k)
