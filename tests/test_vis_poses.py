"""Pose visualisation (gdrnpp_bop2022_b200.vis_poses): the host restatement against the reference's own
vis_object_poses (tests/golden/ref_vis_poses.npz, tools/make_golden_vis_poses.py), the flat-shaded colour renders
against the f64 oracle, the composite kernel against the fixture, and the split CLI end to end."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from gdrnpp_bop2022_b200 import gt_info
from gdrnpp_bop2022_b200 import vis_poses as VP
from gdrnpp_bop2022_b200._lib import GdrnError

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_vis_poses.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _texts(g, i):
    return [[{"name": "", "val": "{}:{}".format(o, k), "fmt": ""}] for k, o in enumerate(g[f"im{i}_obj_ids"])]


def test_host_restatement_matches_reference_fixture(golden):
    g = golden
    for i in (0, 1):
        for resolve in (True, False):
            out = VP.host_vis_object_poses(g[f"im{i}_m_rgb"], g[f"im{i}_m_depth"], g[f"im{i}_rgb"], g[f"im{i}_depth"],
                                           _texts(g, i), resolve_visib=resolve)
            assert np.array_equal(out["rgb"], g[f"im{i}_resolve{int(resolve)}_vis_rgb"]), (i, resolve)
            assert np.array_equal(out["depth_diff"], g[f"im{i}_resolve{int(resolve)}_vis_depth_diff"]), (i, resolve)
    # the fixture covers what it claims: an empty render, equal depths, diffs on both sides of 15 mm
    assert not g["im0_m_rgb"][3].any()
    both = (g["im0_m_depth"][1] > 0) & (g["im0_m_depth"][2] > 0)
    assert both.any() and np.array_equal(g["im0_m_depth"][1][both], g["im0_m_depth"][2][both])
    r = g["im0_resolve1_vis_depth_diff"][12:, :, 0]
    assert (r == 255).any() and (r == 0).any()


def test_depth_for_vis_degenerate_inputs():
    assert not VP.depth_for_vis(np.zeros((2, 3), np.float32)).any()
    x = np.array([[0.0, 2.5], [2.5, 0.0]], np.float32)
    assert np.array_equal((255 * VP.depth_for_vis(x)).astype(np.uint8), [[0, 51], [51, 0]])


def test_cli_parsing():
    a = VP.parse_args(["--dataset", "itodd", "--scene_ids", "1,3", "--im_ids", "5", "--gt_ids", "0,2", "--no_depth_diff",
                       "--renderer_type", "cpp", "--max_bytes", "1000"])
    assert (a.scene_ids, a.im_ids, a.gt_ids, a.no_depth_diff, a.max_bytes) == ([1, 3], [5], [0, 2], True, 1000)
    assert not a.no_vis_rgb and not a.no_resolve_visib and not a.vis_orig_color
    for bad in (["--shading", "phong"], ["--no_vis_rgb", "--no_depth_diff"]):
        with pytest.raises(SystemExit):
            VP.parse_args(bad)


def test_split_image_and_model_paths(tmp_path):
    sp = gt_info.split_params("/d", "itodd", "test")
    assert (sp["im_modality"], sp["im_ext"], sp["depth_ext"]) == ("gray", ".tif", ".tif")
    sp = gt_info.split_params("/d", "lmo", "train", "pbr")
    assert (sp["split_path"], sp["im_modality"], sp["im_ext"]) == ("/d/lmo/train_pbr", "rgb", ".jpg")
    sp = gt_info.split_params("/d", "itodd", "train", "pbr")
    assert (sp["im_modality"], sp["im_ext"]) == ("rgb", ".jpg")
    assert gt_info.split_params("/d", "tless", "test")["im_ext"] == ".png"
    assert gt_info.models_path("/d", "tless", None, "eval") == "/d/tless/models_eval"
    assert gt_info.models_path("/d", "tless") == "/d/tless/models_cad"
    assert gt_info.models_path("/d", "ycbvposecnn", None, "eval") == "/d/ycbv/models_eval"
    sp = gt_info.split_params(str(tmp_path), "lm", "test")
    with pytest.raises(GdrnError, match="missing rgb image"):
        gt_info.image_path(sp, 1, 0)


def _split(root, **kw):
    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    write_bop_tree(root, dataset="ycbv", num_images=5, num_scenes=2, H=48, W=64, dets_per_image=4,
                   obj_ids=[1, 2, 3, 4], **kw)
    return gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "ycbv", "test")


def _models(sp):
    return os.path.join(sp["base_path"], "models_eval")


def test_driver_rejections(tmp_path):
    """Each is rejected, naming the setting or file, before any device work."""
    sp = _split(str(tmp_path / "a"))
    os.remove(os.path.join(_models(sp), "obj_000002.ply"))
    with pytest.raises(GdrnError, match="obj_id 2: no model file"):
        VP.run_split(sp, _models(sp), str(tmp_path / "out"), "ycbv", "test")
    sp = _split(str(tmp_path / "b"))
    os.remove(os.path.join(sp["split_path"], "000001", "rgb", "000001.png"))
    with pytest.raises(GdrnError, match="missing rgb image .*000001.png"):
        VP.run_split(sp, _models(sp), str(tmp_path / "out"), "ycbv", "test")
    sp = _split(str(tmp_path / "c"))
    os.remove(os.path.join(sp["split_path"], "000001", "depth", "000001.png"))
    with pytest.raises(GdrnError, match="missing depth image"):
        VP.run_split(sp, _models(sp), str(tmp_path / "out"), "ycbv", "test")
    sp = _split(str(tmp_path / "d"))
    path = os.path.join(sp["split_path"], "000001", "scene_camera.json")
    with open(path) as f:
        cams = json.load(f)
    del cams[sorted(cams, key=int)[0]]["depth_scale"]
    with open(path, "w") as f:
        json.dump(cams, f)
    with pytest.raises(GdrnError, match="no depth_scale"):
        VP.run_split(sp, _models(sp), str(tmp_path / "out"), "ycbv", "test")
    sp = _split(str(tmp_path / "e"))
    p = os.path.join(_models(sp), "obj_000003.ply")
    with open(p, "rb") as f:
        raw = f.read()
    with open(p, "wb") as f:
        f.write(raw.replace(b"\nelement vertex", b"\ncomment TextureFile obj_000003.png\nelement vertex", 1))
    with pytest.raises(GdrnError, match="obj_id 3: .* is textured; --vis_orig_color"):
        VP.run_split(sp, _models(sp), str(tmp_path / "out"), "ycbv", "test", vis_orig_color=True)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _meshes(dev, with_colors):
    """Two closed meshes in mm: a box and an icosahedron-like blob, one with vertex colours when asked."""
    from gdrnpp_bop2022_b200 import bop_eval

    rs = np.random.RandomState(7)
    box = np.array([[x, y, z] for x in (-30, 30) for y in (-20, 20) for z in (-25, 25)], np.float64)
    bf = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                   [0, 6, 4], [1, 5, 7], [1, 7, 3]])
    t = (1 + 5 ** 0.5) / 2
    ico = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                    [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64) * 18
    icf = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                    [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                    [6, 2, 10], [8, 6, 7], [9, 8, 1]])
    vc = rs.rand(len(ico), 3) if with_colors else None
    return bop_eval.VsdMeshes({1: (box, bf), 2: (ico, icf, vc)}, device=dev), {1: (box, bf, None), 2: (ico, icf, vc)}


def _rot(rs):
    q = rs.randn(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


@pytest.mark.gpu
def test_flat_shading_matches_oracle_and_depth_matches_render_meshes(lib, dev):
    import torch

    from gdrnpp_bop2022_b200 import bop_eval, renderer
    from oracle.flat_shade_oracle import flat_shade

    meshes, host = _meshes(dev, with_colors=True)
    rs = np.random.RandomState(3)
    H, W, n = 60, 80, 8
    obj = [1, 2] * (n // 2)
    R = np.stack([_rot(rs) for _ in range(n)])
    t = np.stack([[rs.uniform(-40, 40), rs.uniform(-30, 30), rs.uniform(300, 600)] for _ in range(n)])
    t[0, :2] = [-250, 0]   # cut by the image border
    K = np.array([[70.0, 0.3, 39.4], [0, 72.0, 30.1], [0, 0, 1]])
    ids = torch.tensor([meshes.ids[o] for o in obj], dtype=torch.int32, device=dev)
    poses = torch.from_numpy(np.concatenate([R, t[:, :, None]], axis=2)).to(dev)
    Ks = torch.from_numpy(np.repeat(K[None], n, 0)).to(dev)
    uni = rs.rand(n, 3)
    for colors in (None, uni):
        rgb, depth, tri = renderer.render_meshes_rgb(ids, poses, Ks, H, W, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR,
                                                     colors=None if colors is None else torch.from_numpy(colors),
                                                     return_tri_ids=True)
        ref_depth = renderer.render_meshes(ids, poses, Ks, H, W, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR, quantize_bits=0)
        assert torch.equal(depth, ref_depth)
        assert torch.equal(tri >= 0, ref_depth > 0)
        rgb, tri = rgb.cpu().numpy(), tri.cpu().numpy()
        for i in range(n):
            v, f, vc = host[obj[i]]
            exp = np.rint(flat_shade(v, f, np.concatenate([R[i], t[i][:, None]], 1), K, tri[i],
                                     None if colors is None else colors[i], vc))
            cov = tri[i] >= 0
            assert cov.any()
            assert np.abs(rgb[i].astype(np.int64) - exp).max() <= 1, (i, colors is None)
            assert not rgb[i][~cov].any()
    # a mesh with neither colours renders grey 0.5 * light_w
    g = renderer.render_meshes_rgb(ids[:1], poses[:1], Ks[:1], H, W, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR)[0][0].cpu()
    on = g.sum(-1) > 0
    assert (g[on][:, 0] == g[on][:, 1]).all() and (g[on][:, 0] >= 64).all() and (g[on][:, 0] <= 128).all()


@pytest.mark.gpu
def test_composite_kernel_reproduces_reference_fixture(lib, dev, golden):
    import torch

    g = golden
    for resolve in (True, False):
        flags = VP.RGB | VP.DEPTH_DIFF | (VP.RESOLVE if resolve else 0)
        m_rgb = torch.from_numpy(np.concatenate([g["im0_m_rgb"], g["im1_m_rgb"]])).to(dev)
        m_depth = torch.from_numpy(np.concatenate([g["im0_m_depth"], g["im1_m_depth"]])).to(dev)
        off = np.array([0, len(g["im0_m_rgb"]), len(g["im0_m_rgb"]) + len(g["im1_m_rgb"])])
        rgb = torch.from_numpy(np.stack([g["im0_rgb"], g["im1_rgb"]])).to(dev)
        depth = torch.from_numpy(np.stack([g["im0_depth"], g["im1_depth"]])).to(dev)
        res = {k: v.cpu().numpy() for k, v in VP.composite_device(m_rgb, m_depth, off, rgb, depth, flags).items()
               if v is not None}
        texts = [_texts(g, 0), _texts(g, 1)]
        outs = VP.finish_host(res, off, texts, flags)
        for i in (0, 1):
            ref = VP.host_vis_object_poses(g[f"im{i}_m_rgb"], g[f"im{i}_m_depth"], g[f"im{i}_rgb"], g[f"im{i}_depth"],
                                           texts[i], resolve_visib=resolve)
            assert [tuple(b) if b else None for b in ref["boxes"]] == [
                (int(b[0]), int(b[1]), int(b[2] - b[0]), int(b[3] - b[1])) if b[0] <= b[2] else None
                for b in res["boxes"][off[i]:off[i + 1]]]
            assert np.array_equal(outs[i]["rgb"], g[f"im{i}_resolve{int(resolve)}_vis_rgb"]), (i, resolve)
            gd = g[f"im{i}_resolve{int(resolve)}_vis_depth_diff"]
            base = res["diff_vis"][i]
            valid = (g[f"im{i}_depth"] > 0) & (res["ren_depth"][i] > 0)
            ren_d = res["ren_depth"][i]
            dv = (ren_d - g[f"im{i}_depth"])[valid]
            assert res["diff_count"][i] == dv.size
            assert res["diff_minmax"][i, 0] == dv.min() and res["diff_minmax"][i, 1] == dv.max()
            assert abs(res["diff_sum"][i] / dv.size - float(np.mean(dv))) < 1e-3
            # every pixel below the three text lines equals the reference; the lines themselves when the printed
            # mean (f64 device sum against NumPy's f32 mean) agrees
            f = VP.font()
            h = sum(f.getbbox(s)[3] for s in ("min diff:0", "max diff:0", "mean diff:0")) + 1
            assert np.array_equal(base[h:], gd[h:]), (i, resolve)
            assert np.array_equal(outs[i]["depth_diff"][h:], gd[h:])
            same_text = "{:.3f}".format(np.float32(res["diff_sum"][i] / dv.size)) == "{:.3f}".format(np.mean(dv))
            if same_text:
                assert np.array_equal(outs[i]["depth_diff"], gd), (i, resolve)


def _read_jpgs(d):
    out = {}
    for root, _, files in os.walk(d):
        for f in sorted(files):
            with open(os.path.join(root, f), "rb") as fh:
                out[os.path.relpath(os.path.join(root, f), d)] = fh.read()
    return out


def _pil_jpg(a):
    from PIL import Image

    b = io.BytesIO()
    Image.fromarray(a).save(b, format="JPEG", quality=95)
    return b.getvalue()


@pytest.mark.gpu
def test_cli_end_to_end_matches_in_memory_and_host_restatement(lib, dev, tmp_path):
    import torch

    from gdrnpp_bop2022_b200 import bop_eval

    root = str(tmp_path / "datasets")
    sp = _split(root)
    colors = os.path.join(str(tmp_path), "colors.json")
    with open(colors, "w") as f:
        json.dump(VP.default_colors()[:7], f)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    outs = []
    for k, mb in enumerate((1 << 30, 200_000, 1 << 30)):
        vis = str(tmp_path / "vis{}".format(k))
        subprocess.run([sys.executable, "-m", "gdrnpp_bop2022_b200.vis_poses", "--dataset", "ycbv", "--dataset_split",
                        "test", "--datasets_path", os.path.join(root, "BOP_DATASETS"), "--vis_path", vis,
                        "--max_bytes", str(mb), "--colors_json", colors, "--renderer_type", "python"],
                       check=True, cwd=str(tmp_path), env=env)
        outs.append(_read_jpgs(vis))
    assert outs[0] and outs[0] == outs[1] == outs[2]
    # the same images in memory, then the host restatement on the library's own renders
    palette = VP.default_colors()[:7]
    images = VP.plan_images(sp)
    used = sorted({int(p["obj_id"]) for im in images for p in im[6]})
    from gdrnpp_bop2022_b200.ply import load_ply

    ms = {o: load_ply(os.path.join(_models(sp), "obj_{:06d}.ply".format(o))) for o in used}
    meshes = bop_eval.VsdMeshes({o: (m["pts"], m["faces"]) for o, m in ms.items()}, device=dev)
    oc = {o: tuple(palette[(o - 1) % len(palette)]) for o in used}
    for scene_id, im_id, K, scale, dpath, ipath, poses in images:
        rgb = VP.read_rgb(ipath)
        depth = gt_info.read_depth(dpath).astype(np.float32) * np.float32(scale)
        o = VP.vis_object_poses(meshes, [poses], K[None], rgb[None], depth[None], obj_colors=oc)[0]
        key = os.path.join("ycbv", "test", "{:06d}".format(scene_id), "{:06d}".format(im_id))
        assert outs[0][key + ".jpg"] == _pil_jpg(o["rgb"])
        assert outs[0][key + "_depth_diff.jpg"] == _pil_jpg(o["depth_diff"])
        m_rgb, m_depth, _ = VP.render_instances(meshes, [poses], K[None], rgb.shape[0], rgb.shape[1], oc)
        ref = VP.host_vis_object_poses(m_rgb.cpu().numpy(), m_depth.cpu().numpy(), rgb, depth,
                                       [p["text_info"] for p in poses])
        assert np.array_equal(o["rgb"], ref["rgb"])
        f = VP.font()
        h = sum(f.getbbox(s)[3] for s in ("min diff:0", "max diff:0", "mean diff:0")) + 1
        assert np.array_equal(o["depth_diff"][h:], ref["depth_diff"][h:])
        torch.cuda.synchronize()


def test_no_vis_rgb_needs_no_colour_images(tmp_path):
    sp = _split(str(tmp_path / "a"))
    os.remove(os.path.join(sp["split_path"], "000001", "rgb", "000001.png"))
    images = VP.plan_images(sp, rgb_vis=False)
    assert images and all(im[5] is None for im in images)
    with pytest.raises(GdrnError, match="missing rgb image"):
        VP.plan_images(sp)


@pytest.mark.gpu
def test_result_csv_draws_the_estimates(lib, dev, tmp_path):
    from gdrnpp_bop2022_b200 import bop_eval
    from gdrnpp_bop2022_b200.ply import load_ply

    root = str(tmp_path / "datasets")
    sp = _split(root)
    images = VP.plan_images(sp)
    scene_id, im_id, K, scale, dpath, ipath, poses = images[0]
    rs = np.random.RandomState(5)
    csv = str(tmp_path / "gdrn_ycbv-test.csv")
    with open(csv, "w") as f:   # estimates: the GT poses moved and turned, so drawing GT instead would differ
        f.write("scene_id,im_id,obj_id,score,R,t,time\n")
        for k, p in enumerate(poses[:2]):
            R = _rot(rs) @ np.asarray(p["R"]).reshape(3, 3) if k == 0 else np.asarray(p["R"]).reshape(3, 3)
            t = np.asarray(p["t"], np.float64).ravel() + [15.0, -10.0, 30.0]
            f.write("{},{},{},{},{},{},0.1\n".format(scene_id, im_id, p["obj_id"], 0.875 - 0.25 * k,
                                                     " ".join("%.9g" % v for v in R.ravel()),
                                                     " ".join("%.9g" % v for v in t)))
    vis = str(tmp_path / "vis")
    VP.main(["--dataset", "ycbv", "--dataset_split", "test", "--datasets_path", os.path.join(root, "BOP_DATASETS"),
             "--vis_path", vis, "--result_filename", csv, "--scene_ids", str(scene_id), "--im_ids", str(im_id)])
    out = os.path.join(vis, "gdrn_ycbv-test", "ycbv", "test", "{:06d}".format(scene_id), "{:06d}".format(im_id))
    # the same estimates, in file order with "{obj_id}:{score:.2f}", through the in-memory API
    rows = [{"obj_id": r["obj_id"], "R": r["R"], "t": r["t"],
             "text_info": [{"name": "", "val": "{}:{:.2f}".format(r["obj_id"], r["score"]), "fmt": ""}]}
            for r in bop_eval.load_bop_results(csv)]
    assert [r["text_info"][0]["val"] for r in rows] == ["{}:0.88".format(poses[0]["obj_id"]),
                                                         "{}:0.62".format(poses[1]["obj_id"])]
    used = sorted({r["obj_id"] for r in rows})
    ms = {o: load_ply(os.path.join(_models(sp), "obj_{:06d}.ply".format(o))) for o in used}
    meshes = bop_eval.VsdMeshes({o: (m["pts"], m["faces"]) for o, m in ms.items()}, device=dev)
    pal = VP.default_colors()
    oc = {o: tuple(pal[(o - 1) % len(pal)]) for o in used}
    rgb = VP.read_rgb(ipath)
    depth = gt_info.read_depth(dpath).astype(np.float32) * np.float32(scale)
    o = VP.vis_object_poses(meshes, [rows], K[None], rgb[None], depth[None], obj_colors=oc)[0]
    with open(out + ".jpg", "rb") as f:
        assert f.read() == _pil_jpg(o["rgb"])
    with open(out + "_depth_diff.jpg", "rb") as f:
        assert f.read() == _pil_jpg(o["depth_diff"])
    gt = VP.vis_object_poses(meshes, [[dict(p) for p in poses[:2]]], K[None], rgb[None], depth[None], obj_colors=oc)[0]
    assert not np.array_equal(gt["rgb"], o["rgb"])


def _restated_demo_panels(image, masks, boxes, names, pts, K, cur_res):
    """predictor_gdrn.py:583-630 in the reference's own per-element form (misc.project_pts, the per-point
    misc.points2d_to_mask loop, vis_utils.image's blends with colours drawn from np.random), with ROI i's own object."""
    import cv2

    def blend(img, mask, color):
        m = mask.astype(bool)
        img[m] = img[m] * 0.5 + color * 0.5

    H, W = image.shape[:2]
    panels = []
    im = image.copy()
    for i, mask in enumerate(masks):
        blend(im, mask, np.random.randint(0, 256, (1, 3), dtype=np.uint8))
        x1, y1, x2, y2 = boxes[i].astype(np.int32)[:4]
        cv2.rectangle(im, (int(x1), int(y1)), (int(x2), int(y2)), (18, 127, 15), thickness=1)
        cv2.putText(im, names[i], (int(x1), max(int(y1) - 2, 5)), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (0, 255, 0), 2)
    panels.append(im[:, :, ::-1])
    for i, res in enumerate(cur_res):
        P = K.dot(np.hstack((res["R"], res["t"].reshape(3, 1))))
        p = P.dot(np.hstack((pts[i], np.ones((pts[i].shape[0], 1)))).T)
        p /= p[2, :]
        mask = np.zeros((H, W), np.uint8)
        for x, y in p[:2, :].T:
            x, y = int(round(x)), int(round(y))
            if 0 <= x < W and 0 <= y < H:
                mask[y, x] = 1
        im = image.copy()
        blend(im, mask, np.array((0, 255, 255) if i == 0 else (255, 0, 0), np.uint8))
        x1, y1, x2, y2 = boxes[i].astype(np.int32)[:4]
        cv2.rectangle(im, (int(x1), int(y1)), (int(x2), int(y2)), (18, 127, 15), thickness=2)
        cv2.putText(im, names[i], (int(x1), int(y1) - 2), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (0, 255, 0), 2)
        panels.append(im[:, :, ::-1])
    return np.hstack([cv2.cvtColor(v, cv2.COLOR_BGR2RGB) for v in panels])


@pytest.mark.gpu
def test_demo_loop_ends_with_gdrn_visualization(lib, dev):
    """demo_gdrn.py's loop: YoloPredictor -> preprocessing -> inference -> postprocessing -> gdrn_visualization."""
    from types import SimpleNamespace

    import torch

    from gdrnpp_bop2022_b200 import native_ops
    from gdrnpp_bop2022_b200.gdrn_model import _cfg_get
    from gdrnpp_bop2022_b200.predictor import GdrnPredictor
    from gdrnpp_bop2022_b200.predictor_yolo import YoloPredictor
    from gdrnpp_bop2022_b200.synthetic import YCBV_K, make_state_dict, make_yolox_state_dict
    from gdrnpp_bop2022_b200.renderer import get_out_mask
    from oracle import yolox_oracle

    sd = make_yolox_state_dict(yolox_oracle.yolox_forward, 0.33, 0.25, 3, seed=0, calib_hw=(640, 640), calib_batch=2,
                               device="cuda")
    yolo = YoloPredictor(cfg=SimpleNamespace(depth=0.33, width=0.25, num_classes=3, test_size=(640, 640), conf_thr=0.3,
                                             nms_thr=0.65), state_dict=sd)
    objs = {i: "obj_%06d" % i for i in range(1, 22)}
    box = np.array([[x, y, z] for x in (-0.05, 0.05) for y in (-0.04, 0.04) for z in (-0.03, 0.03)], np.float32)
    faces = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                      [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    models = {i: (box * (1 + 0.05 * i), faces) for i in objs}
    gdrn = GdrnPredictor(cam=YCBV_K, objs=objs, extents={i: np.ptp(models[i][0], axis=0) for i in objs},
                         models=models, state_dict=make_state_dict())
    img = (np.random.RandomState(2).rand(480, 640, 3) * 255).astype(np.uint8)
    outputs = yolo.inference(img)
    assert outputs[0] is not None
    data = gdrn.preprocessing(outputs=outputs, image=img)
    out = gdrn.inference(data)
    gdrn.postprocessing(data, out)
    n = data["roi_img"].shape[0]
    assert n >= 1 and "full_mask" in out
    np.random.seed(123)
    got = gdrn.gdrn_visualization(batch=data, out_dict=out, image=img, show=False)
    assert got.shape == (480, 640 * (n + 1), 3) and got.dtype == np.uint8
    half = data["scale"].view(n, -1) / 2
    rois = torch.cat([data["roi_center"] - half, data["roi_center"] + half], dim=1)
    loss_type = str(_cfg_get(gdrn.cfg, "MODEL.POSE_NET.LOSS_CFG.MASK_LOSS_TYPE", "L1"))
    masks = native_ops.paste_masks_in_image(get_out_mask(out["full_mask"], loss_type)[:, 0], rois, (480, 640), 0.5)
    masks = masks.to(torch.uint8).cpu().numpy()
    assert masks.any()
    ids = [gdrn.obj_ids[int(c)] for c in data["roi_cls"].tolist()]
    np.random.seed(123)
    exp = _restated_demo_panels(img, masks, [np.asarray(b) for b in data["bbox_est"]], [objs[o] for o in ids],
                                [models[o][0].astype(np.float64) for o in ids], gdrn.cam.astype(np.float64),
                                data["cur_res"])
    assert np.array_equal(got, exp)
    # no detections: the image itself, as the full-mask panel with nothing pasted
    yolo.cfg.conf_thr = 1.01
    data = gdrn.preprocessing(outputs=yolo.inference(img), image=img)
    empty = {"full_mask": torch.zeros((0, 1, 64, 64), device=dev)}
    assert np.array_equal(gdrn.gdrn_visualization(data, empty, img, show=False), img)
