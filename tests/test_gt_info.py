"""Ground-truth annotations of a BOP split (gdrnpp_bop2022_b200/gt_info.py, csrc/gt_info.cu).

The CPU tests pin the host restatement of calc_gt_info.py / calc_gt_masks.py and the JSON writer to
tests/golden/ref_gt_info.npz (written by tools/make_golden_gt_info.py from the reference's own code), and check the
split layout and the driver's rejections.  The GPU tests hold the kernel to the fixture bit for bit and the whole
driver to the host restatement run on the library's own renders."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from gdrnpp_bop2022_b200 import gt_info
from gdrnpp_bop2022_b200._lib import GdrnError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_gt_info.npz")
FIELDS = ("px_count_all", "px_count_valid", "px_count_visib", "visib_fract", "bbox_obj", "bbox_visib")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _test_depth_mm(g, i):
    d = g["depth_test"][i].astype(np.float32)
    d *= g["depth_scale"][i]
    return d


# ---------------------------------------------------------------------------------------------------------------------
# CPU
def test_host_restatement_matches_reference_fixture(golden):
    g = golden
    for i, img in enumerate(g["inst_img"]):
        info, mask, mask_visib = gt_info.host_annotation(g["depth_large"][i], g["depth_img"][i], _test_depth_mm(g, img),
                                                         g["K"][img], float(g["delta"]))
        for k in FIELDS:
            assert np.array_equal(np.asarray(info[k]), g[k][i]), (i, k)
        assert np.array_equal(mask, g["mask"][i]) and np.array_equal(mask_visib, g["mask_visib"][i]), i
    # the cases the fixture is built to hold
    assert list(g["bbox_obj"][1][:1]) == [-6] and list(g["bbox_obj"][2]) == [-1] * 4 and g["px_count_all"][2] > 0
    assert g["px_count_visib"][3] == 0 and g["px_count_valid"][3] > 0 and g["px_count_all"][4] == 0
    assert g["px_count_valid"][5] == 0 and g["visib_fract"][5] == 1.0


def test_json_writer_reproduces_reference_bytes(golden, tmp_path):
    content = {int(k): v for k, v in json.loads(golden["save_json_content"].tobytes().decode()).items()}
    path = str(tmp_path / "scene_gt_info.json")
    gt_info.save_json(path, dict(sorted(content.items())))
    with open(path, "rb") as f:
        assert f.read() == golden["save_json_bytes"].tobytes()
    gt_info.save_json(path, {})
    with open(path, "rb") as f:
        assert f.read() == b"{\n}"


def test_calc_2d_bbox_has_no_plus_one():
    assert gt_info.calc_2d_bbox(np.array([3, 7, 5]), np.array([-2, 4, 0])) == [3, -2, 4, 6]
    assert gt_info.calc_2d_bbox(np.array([9]), np.array([1])) == [9, 1, 0, 0]


def test_split_model_and_depth_resolution(tmp_path):
    r = str(tmp_path)
    sp = gt_info.split_params(r, "lm", "test")
    assert sp["split_path"] == os.path.join(r, "lm", "test") and sp["depth_ext"] == ".png"
    assert gt_info.split_params(r, "lmo", "train", "pbr")["split_path"] == os.path.join(r, "lmo", "train_pbr")
    assert gt_info.split_params(r, "tless", "test")["split_path"] == os.path.join(r, "tless", "test_primesense")
    assert gt_info.split_params(r, "tless", "train", "render_reconst")["split_path"] == os.path.join(
        r, "tless", "train_render_reconst")
    assert gt_info.split_params(r, "hb", "val")["split_path"] == os.path.join(r, "hb", "val_primesense")
    assert gt_info.split_params(r, "hbs", "test", "kinect")["split_path"] == os.path.join(r, "hb", "test_kinect")
    assert gt_info.split_params(r, "ycbv", "train")["split_path"] == os.path.join(r, "ycbv", "train_real")
    assert gt_info.split_params(r, "ycbvposecnn", "test")["split_path"] == os.path.join(r, "ycbv", "test")
    assert gt_info.split_params(r, "tudl", "train")["split_path"] == os.path.join(r, "tudl", "train_render")
    assert gt_info.split_params(r, "lm", "train", "bb8")["split_path"] == os.path.join(r, "lm", "train")
    assert gt_info.split_params(r, "itodd", "val")["depth_ext"] == ".tif"
    with pytest.raises(ValueError, match="Unknown BOP dataset"):
        gt_info.split_params(r, "nope", "test")
    assert gt_info.models_path(r, "lm") == os.path.join(r, "lm", "models")
    assert gt_info.models_path(r, "tless") == os.path.join(r, "tless", "models_cad")
    assert gt_info.models_path(r, "hbs") == os.path.join(r, "hb", "models")
    assert gt_info.models_path(r, "tless", "/x/models_reconst") == "/x/models_reconst"
    # depth: the split's extension, .tif falling back to .png
    sp = gt_info.split_params(r, "itodd", "val")
    os.makedirs(os.path.join(sp["split_path"], "000001", "depth"))
    os.makedirs(os.path.join(sp["split_path"], "000003"))
    os.makedirs(os.path.join(sp["split_path"], "notes"))
    png = os.path.join(sp["split_path"], "000001", "depth", "000004.png")
    open(png, "w").close()
    assert gt_info.depth_path(sp["split_path"], 1, 4, ".tif") == png
    tif = png[:-4] + ".tif"
    open(tif, "w").close()
    assert gt_info.depth_path(sp["split_path"], 1, 4, ".tif") == tif
    assert gt_info.present_scene_ids(sp["split_path"]) == [1, 3]


def test_cli_parsing():
    a = gt_info.parse_args(["--dataset", "tless", "--dataset_split", "train", "--dataset_split_type", "pbr", "--delta",
                            "5", "--what", "masks", "--scene_ids", "3,1", "--max_bytes", "1000", "--renderer_type", "cpp"])
    assert a.dataset == "tless" and a.dataset_split_type == "pbr" and a.delta == 5.0 and a.what == ["masks"]
    assert a.scene_ids == [3, 1] and a.max_bytes == 1000
    d = gt_info.parse_args([])
    assert d.what == ["info", "masks"] and d.delta == 15.0 and d.scene_ids is None
    with pytest.raises(SystemExit):
        gt_info.parse_args(["--what", "info,coco"])


def _tiny_tree(root, H=12, W=16, sizes=None, drop_scale=False, drop_depth=False, obj_ids=(1, 2)):
    """One scene of three images (the middle one without instances) and box models for obj 1 only."""
    import cv2

    from gdrnpp_bop2022_b200.ply import save_ply

    sp = gt_info.split_params(root, "lm", "test")
    sdir = os.path.join(sp["split_path"], "000002")
    os.makedirs(os.path.join(sdir, "depth"))
    models = os.path.join(root, "lm", "models")
    os.makedirs(models)
    pts = np.array([[x, y, z] for x in (-20, 20) for y in (-20, 20) for z in (-20, 20)], np.float32)
    faces = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                      [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    save_ply(os.path.join(models, "obj_000001.ply"), pts, faces)
    gts, cams = {}, {}
    for k, im in enumerate((0, 1, 2)):
        gts[str(im)] = [] if im == 1 else [{"obj_id": int(o), "cam_R_m2c": np.eye(3).ravel().tolist(),
                                            "cam_t_m2c": [0.0, 0.0, 500.0]} for o in obj_ids]
        cams[str(im)] = {"cam_K": [20.0, 0, W / 2, 0, 20.0, H / 2, 0, 0, 1]}
        if not (drop_scale and im == 2):
            cams[str(im)]["depth_scale"] = 1.0
        h, w = (sizes or {}).get(im, (H, W))
        if not (drop_depth and im == 2):
            cv2.imwrite(os.path.join(sdir, "depth", "{:06d}.png".format(im)), np.full((h, w), 900, np.uint16))
    for name, c in (("scene_gt.json", gts), ("scene_camera.json", cams)):
        with open(os.path.join(sdir, name), "w") as f:
            json.dump(c, f)
    return sp, models


def test_driver_rejections(tmp_path):
    sp, models = _tiny_tree(str(tmp_path / "a"))
    with pytest.raises(GdrnError, match=r"obj_id 2: no model file .*obj_000002\.ply"):
        gt_info.run_split(sp, models)
    sp, models = _tiny_tree(str(tmp_path / "b"), obj_ids=(1,), drop_depth=True)
    with pytest.raises(GdrnError, match=r"missing depth image .*000002[/\\]depth[/\\]000002\.png"):
        gt_info.run_split(sp, models)
    sp, models = _tiny_tree(str(tmp_path / "c"), obj_ids=(1,), drop_scale=True)
    with pytest.raises(GdrnError, match="scene 2 image 2: scene_camera.json has no depth_scale"):
        gt_info.run_split(sp, models)
    sp, models = _tiny_tree(str(tmp_path / "d"), obj_ids=(1,), sizes={2: (12, 18)})
    with pytest.raises(GdrnError, match=r"depth image .*000002\.png is 18x12, other images of scene 2 are 16x12"):
        gt_info.run_split(sp, models)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _kernel(lib, dev, g, idx, with_large=True, with_img=True):
    import torch

    from gdrnpp_bop2022_b200 import _lib

    n, (N, H, W) = len(idx), g["depth_test"].shape
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    dl = t(g["depth_large"][idx]) if with_large else None
    di = t(g["depth_img"][idx]) if with_img else None
    dt = t(g["depth_test"].view(np.int16))
    counts = torch.full((n, 3), -7, dtype=torch.int64, device=dev)
    boxes = torch.full((n, 8), -7, dtype=torch.int32, device=dev)
    mask = torch.full((n, H, W), 7, dtype=torch.uint8, device=dev)
    mv = torch.full((n, H, W), 7, dtype=torch.uint8, device=dev)
    scale, K, img = t(g["depth_scale"].astype(np.float32)), t(g["K"].astype(np.float64)), t(g["inst_img"][idx].astype(np.int32))
    _lib.check(lib.gdrn_gt_info(_lib.ptr(dl), _lib.ptr(di), _lib.ptr(dt), _lib.ptr(scale), _lib.ptr(K), _lib.ptr(img), n,
                                H, W, float(g["delta"]), _lib.ptr(counts), _lib.ptr(boxes), _lib.ptr(mask), _lib.ptr(mv),
                                _lib.current_stream()), "gdrn_gt_info")
    return counts.cpu().numpy(), boxes.cpu().numpy(), mask.cpu().numpy(), mv.cpu().numpy()


@pytest.mark.gpu
def test_kernel_matches_reference_fixture_bit_exact(lib, dev, golden):
    g = golden
    n = len(g["inst_img"])
    for idx in (np.arange(n), np.arange(n)[::-1].copy(), np.array([3])):
        counts, boxes, mask, mv = _kernel(lib, dev, g, idx)
        assert np.array_equal(counts[:, 0], g["px_count_all"][idx])
        assert np.array_equal(counts[:, 1], g["px_count_valid"][idx])
        assert np.array_equal(counts[:, 2], g["px_count_visib"][idx])
        assert np.array_equal(boxes[:, :4], g["bbox_obj"][idx]) and np.array_equal(boxes[:, 4:], g["bbox_visib"][idx])
        assert np.array_equal(mask, g["mask"][idx]) and np.array_equal(mv, g["mask_visib"][idx])
        with np.errstate(invalid="ignore", divide="ignore"):
            vf = np.where(counts[:, 0] > 0, counts[:, 2] / counts[:, 0].astype(np.float64), 0.0)
        assert np.array_equal(vf, g["visib_fract"][idx])
    # info only (no masks written) and masks only (no canvas: counts 0, boxes -1)
    counts, boxes, mask, _ = _kernel(lib, dev, g, np.arange(n), with_img=False)
    assert np.array_equal(counts[:, 2], g["px_count_visib"]) and (mask == 7).all()
    counts, boxes, mask, mv = _kernel(lib, dev, g, np.arange(n), with_large=False)
    assert (counts == 0).all() and (boxes == -1).all()
    assert np.array_equal(mask, g["mask"]) and np.array_equal(mv, g["mask_visib"])


def _box_meshes():
    faces = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                      [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    out = {}
    for o, half in {1: (30.0, 20.0, 15.0), 2: (25.0, 25.0, 40.0)}.items():
        out[o] = (np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32) * half, faces)
    return out


def _host_renders(meshes, obj_ids, R, t, K, H, W):
    """The library's own renders at both canvases, as annotate_device makes them."""
    import torch

    from gdrnpp_bop2022_b200 import bop_eval, renderer

    n = len(obj_ids)
    dev = meshes.device
    ids = torch.tensor([meshes.ids[int(o)] for o in obj_ids], dtype=torch.int32, device=dev)
    poses = torch.from_numpy(np.concatenate([np.asarray(R, np.float64).reshape(n, 3, 3),
                                             np.asarray(t, np.float64).reshape(n, 3, 1)], axis=2)).to(dev)
    K = np.asarray(K, np.float64).reshape(n, 3, 3)
    KL = K.copy()
    KL[:, 0, 2] += W
    KL[:, 1, 2] += H
    large = renderer.render_meshes(ids, poses, torch.from_numpy(KL).to(dev), 3 * H, 3 * W, bop_eval.VSD_ZNEAR,
                                   bop_eval.VSD_ZFAR, quantize_bits=0)
    img = renderer.render_meshes(ids, poses, torch.from_numpy(K).to(dev), H, W, bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR,
                                 quantize_bits=0)
    return large.cpu().numpy(), img.cpu().numpy()


@pytest.mark.gpu
def test_in_memory_edge_cases_and_chunking_on_vsd_meshes(lib, dev):
    from gdrnpp_bop2022_b200 import bop_eval

    H, W = 120, 160
    meshes = bop_eval.VsdMeshes(_box_meshes(), device=dev)
    K = np.array([[[150.0, 0, 80.3], [0, 150.0, 59.6], [0, 0, 1]], [[140.0, 0, 77.0], [0, 145.0, 62.0], [0, 0, 1]],
                  [[150.0, 0, 80.0], [0, 150.0, 60.0], [0, 0, 1]]])
    yy, xx = np.mgrid[0:H, 0:W]
    plane = np.round(800 + 200 * xx / W + 50 * yy / H).astype(np.uint16)
    depth = np.stack([plane, np.zeros((H, W), np.uint16), plane // 2])   # image 1: no sensor depth at all
    scale = [1.0, 0.1, 2.0]
    R = np.stack([np.eye(3)] * 6)
    t = np.array([[0.0, 0, 700],      # in front of the plane: visible
                  [-300.0, 10, 600],  # partly outside the image (left): negative bbox_obj
                  [1000.0, 0, 600],   # outside the image, inside the canvas: -1 boxes
                  [0.0, 0, 1200],     # behind the plane: fully occluded
                  [10.0, -5, 900],    # image 1: missing depth, visible under bop19
                  [0.0, 0, 600]])     # image 2
    obj = [1, 2, 1, 2, 1, 2]
    img = [0, 0, 0, 0, 1, 2]
    ref = gt_info.annotate(meshes, obj, R, t, img, K, depth, scale, masks=True)
    assert ref["bbox_obj"][1][0] < 0 and ref["px_count_visib"][1] > 0
    assert list(ref["bbox_obj"][2]) == [-1] * 4 and ref["px_count_all"][2] > 0 and ref["visib_fract"][2] == 0.0
    assert ref["px_count_visib"][3] == 0 and ref["px_count_valid"][3] > 0 and list(ref["bbox_visib"][3]) == [-1] * 4
    assert ref["px_count_valid"][4] == 0 and ref["visib_fract"][4] == 1.0
    large, small = _host_renders(meshes, obj, R, t, K[img], H, W)
    for i in range(len(obj)):
        dmm = depth[img[i]].astype(np.float32)
        dmm *= scale[img[i]]
        info, m, mv = gt_info.host_annotation(large[i], small[i], dmm, K[img[i]], 15)
        for k in FIELDS:
            assert np.array_equal(np.asarray(info[k]), ref[k][i]), (i, k)
        assert np.array_equal(m, ref["mask"][i]) and np.array_equal(mv, ref["mask_visib"][i]), i
    # chunking, order of the calls and a second run change nothing
    for mb in (1, gt_info.instance_bytes(H, W) * 2 + 5, 1 << 40):
        got = gt_info.annotate(meshes, obj, R, t, img, K, depth, scale, masks=True, max_bytes=mb)
        assert all(np.array_equal(got[k], ref[k]) for k in ref), mb
    only_info = gt_info.annotate(meshes, obj, R, t, img, K, depth, scale)
    assert all(np.array_equal(only_info[k], ref[k]) for k in FIELDS) and "mask" not in only_info
    only_masks = gt_info.annotate(meshes, obj, R, t, img, K, depth, scale, masks=True, info=False)
    assert np.array_equal(only_masks["mask"], ref["mask"]) and np.array_equal(only_masks["mask_visib"], ref["mask_visib"])
    empty = gt_info.annotate(meshes, [], R[:0], t[:0], [], K, depth, scale, masks=True)
    assert empty["px_count_all"].shape == (0,) and empty["mask"].shape == (0, H, W)


def _synthetic_split(root):
    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    write_bop_tree(root, dataset="ycbv", num_images=7, num_scenes=2, dets_per_image=5, obj_ids=[1, 2, 3, 4, 5, 6])
    base = os.path.join(root, "BOP_DATASETS", "ycbv")
    shutil.copytree(os.path.join(base, "models_eval"), os.path.join(base, "models"))
    # an image without instances
    sp = gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "ycbv", "test")
    path = os.path.join(sp["split_path"], "000002", "scene_gt.json")
    with open(path) as f:
        gts = json.load(f)
    gts[sorted(gts, key=int)[1]] = []
    with open(path, "w") as f:
        json.dump(gts, f)
    return sp


def _read_outputs(sp):
    import cv2

    out = {}
    for s in gt_info.present_scene_ids(sp["split_path"]):
        sdir = os.path.join(sp["split_path"], "{:06d}".format(s))
        with open(os.path.join(sdir, "scene_gt_info.json"), "rb") as f:
            out[(s, "json")] = f.read()
        for d in ("mask", "mask_visib"):
            for name in sorted(os.listdir(os.path.join(sdir, d))):
                out[(s, d, name)] = cv2.imread(os.path.join(sdir, d, name), cv2.IMREAD_UNCHANGED)
    return out


@pytest.mark.gpu
def test_cli_end_to_end_matches_host_restatement_on_vsd_meshes(lib, dev, tmp_path):
    from gdrnpp_bop2022_b200 import bop_eval

    root = str(tmp_path / "datasets")
    sp = _synthetic_split(root)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    subprocess.run([sys.executable, "-m", "gdrnpp_bop2022_b200.gt_info", "--dataset", "ycbv", "--dataset_split", "test",
                    "--datasets_path", os.path.join(root, "BOP_DATASETS"), "--renderer_type", "python"],
                   check=True, cwd=str(tmp_path), env=env)
    got = _read_outputs(sp)
    models = gt_info.load_models(gt_info.models_path(os.path.join(root, "BOP_DATASETS"), "ycbv"), range(1, 7))
    meshes = bop_eval.VsdMeshes(models, device=dev)
    n_vis = n_occ = 0
    for scene_id, ims in gt_info.plan_split(sp):
        scene_info = {}
        for im in ims:
            depth = gt_info.read_depth(im["depth"]).astype(np.float32)
            depth *= im["depth_scale"]
            H, W = depth.shape
            gts = im["gts"]
            recs = []
            if gts:
                large, small = _host_renders(meshes, [g["obj_id"] for g in gts], [g["cam_R_m2c"] for g in gts],
                                             [g["cam_t_m2c"] for g in gts], [im["K"]] * len(gts), H, W)
            for j, g in enumerate(gts):
                info, m, mv = gt_info.host_annotation(large[j], small[j], depth, im["K"], 15)
                recs.append(info)
                n_vis += 0 < info["visib_fract"] < 1
                n_occ += info["px_count_visib"] < info["px_count_all"]
                name = "{:06d}_{:06d}.png".format(im["im_id"], j)
                assert np.array_equal(got[(scene_id, "mask", name)], m), name
                assert np.array_equal(got[(scene_id, "mask_visib", name)], mv), name
            scene_info[im["im_id"]] = recs
        path = str(tmp_path / "host.json")
        gt_info.save_json(path, scene_info)
        with open(path, "rb") as f:
            assert f.read() == got[(scene_id, "json")], scene_id
    assert n_vis > 0 and n_occ > 0
    assert b": []" in got[(2, "json")]


@pytest.mark.gpu
def test_driver_outputs_identical_across_batching_and_runs(lib, dev, tmp_path):
    root = str(tmp_path / "datasets")
    sp = _synthetic_split(root)
    models = gt_info.models_path(os.path.join(root, "BOP_DATASETS"), "ycbv")
    runs = []
    for kw in ({}, {"batch_images": 1}, {"batch_images": 3, "max_bytes": 1}, {"max_bytes": 40 << 20}, {}):
        r = gt_info.run_split(sp, models, device=dev, **kw)
        assert r["images"] == 7 and r["instances"] == 30
        runs.append(_read_outputs(sp))
    for o in runs[1:]:
        assert o.keys() == runs[0].keys()
        for k in o:
            assert np.array_equal(np.frombuffer(o[k], np.uint8) if isinstance(o[k], bytes) else o[k],
                                  np.frombuffer(runs[0][k], np.uint8) if isinstance(runs[0][k], bytes) else runs[0][k]), k
    # one part at a time writes the same files
    shutil.rmtree(os.path.join(sp["split_path"], "000001", "mask"))
    gt_info.run_split(sp, models, what=("masks",), scene_ids=[1], device=dev)
    gt_info.run_split(sp, models, what=("info",), device=dev)
    o = _read_outputs(sp)
    assert all(np.array_equal(np.frombuffer(o[k], np.uint8) if isinstance(o[k], bytes) else o[k],
                              np.frombuffer(runs[0][k], np.uint8) if isinstance(runs[0][k], bytes) else runs[0][k])
               for k in runs[0])
