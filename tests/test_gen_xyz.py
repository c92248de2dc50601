"""xyz_crop training targets of a BOP split (gdrnpp_bop2022_b200/gen_xyz.py, csrc/xyz_crop.cu).

The CPU tests check the CLI, the split / model / output layout the reference's *_1_gen_xyz.py scripts hard-code, the
resume plan, the driver's refusals and the fp64 oracle (oracle/xyz_crop_oracle.py) against a restatement of
misc.calc_xyz_bp_torch in f32 torch.  The GPU tests hold the kernels to the oracle on BOP-scale meshes, the pass's
renders to the EGLRenderer surface bit for bit, and the split driver's files to the oracle's bytes."""
import json
import os
import pickle
import shutil
import subprocess
import sys

import numpy as np
import pytest

from gdrnpp_bop2022_b200 import gen_xyz, gt_info
from gdrnpp_bop2022_b200._lib import GdrnError
from oracle import xyz_crop_oracle as XO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------
# CPU
def test_cli_parsing():
    a = gen_xyz.parse_args(["--dataset", "tless", "--dataset_split", "train", "--dataset_split_type", "pbr",
                            "--datasets_path", "/d", "--xyz_root", "/o", "--scene_ids", "3,1", "--max_bytes", "1000",
                            "--batch_images", "4"])
    assert a.dataset == "tless" and a.dataset_split == "train" and a.dataset_split_type == "pbr"
    assert a.datasets_path == "/d" and a.xyz_root == "/o" and a.scene_ids == [3, 1] and a.max_bytes == 1000
    assert a.batch_images == 4 and a.models_dir is None and a.model_type is None
    d = gen_xyz.parse_args(["--dataset", "icbin"])
    assert d.dataset_split == "train" and d.scene_ids is None and d.max_bytes == gen_xyz.DEFAULT_MAX_BYTES
    with pytest.raises(SystemExit):
        gen_xyz.parse_args([])
    with pytest.raises(SystemExit):
        gen_xyz.parse_args(["--dataset", "tless", "--models_dir", "/m", "--model_type", "reconst"])


@pytest.mark.parametrize("script,argv,split,models", [
    ("icbin_pbr_1_gen_xyz.py", ["--dataset", "icbin", "--dataset_split", "train", "--dataset_split_type", "pbr"],
     "icbin/train_pbr", "icbin/models"),
    ("itodd_pbr_1_gen_xyz.py", ["--dataset", "itodd", "--dataset_split", "train", "--dataset_split_type", "pbr"],
     "itodd/train_pbr", "itodd/models"),
    ("tudl_pbr_1_gen_xyz.py", ["--dataset", "tudl", "--dataset_split", "train", "--dataset_split_type", "pbr"],
     "tudl/train_pbr", "tudl/models"),
    ("tless_pbr_1_gen_xyz.py", ["--dataset", "tless", "--dataset_split", "train", "--dataset_split_type", "pbr"],
     "tless/train_pbr", "tless/models_cad"),
    ("tless_primesense_1_gen_xyz.py", ["--dataset", "tless", "--dataset_split", "train", "--dataset_split_type",
                                       "primesense_rescaled", "--model_type", "reconst"],
     "tless/train_primesense_rescaled", "tless/models_reconst"),
    ("(no script) lmo train_pbr", ["--dataset", "lmo", "--dataset_split", "train", "--dataset_split_type", "pbr"],
     "lmo/train_pbr", "lmo/models"),
])
def test_reference_scripts_resolve_to_their_directories(script, argv, split, models):
    root = os.path.join(os.sep, "data", "BOP_DATASETS")
    sp, model_dir, xyz_root = gen_xyz.resolve(gen_xyz.parse_args(argv + ["--datasets_path", root]))
    assert sp["split_path"] == os.path.join(root, *split.split("/")), script
    assert model_dir == os.path.join(root, *models.split("/")), script
    assert xyz_root == os.path.join(root, *split.split("/"), "xyz_crop"), script
    a = gen_xyz.parse_args(argv + ["--datasets_path", root, "--xyz_root", "/x", "--models_dir", "/m"]
                           if "--model_type" not in argv else argv + ["--datasets_path", root, "--xyz_root", "/x"])
    assert gen_xyz.resolve(a)[2] == "/x"


def test_path_layout():
    assert gen_xyz.xyz_path("/r/xyz_crop", 3, 17, 5) == os.path.join("/r/xyz_crop", "000003", "000017_000005-xyz.pkl")


def _tree(root, **kw):
    from gdrnpp_bop2022_b200.synthetic import write_bop_train_tree

    base = write_bop_train_tree(root, dataset="lmo", num_images=6, num_scenes=2, H=48, W=64, insts_per_image=3, num_bg=1,
                                **kw)
    sp = gt_info.split_params(os.path.join(root, "BOP_DATASETS"), "lmo", "train", "pbr")
    return sp, os.path.join(base, "models")


def _edit_json(path, fn):
    with open(path) as f:
        c = json.load(f)
    fn(c)
    with open(path, "w") as f:
        json.dump(c, f)


def test_resume_plan(tmp_path):
    sp, _ = _tree(str(tmp_path))
    xyz_root = os.path.join(sp["split_path"], "xyz_crop")
    scenes, skipped = gen_xyz.plan(sp, xyz_root)
    assert skipped == 0 and [s[0] for s in scenes] == [0, 1] and all(s[1] == (48, 64) for s in scenes)
    assert sum(len(insts) for s in scenes for _, insts in s[2]) == 18 and sum(s[3] for s in scenes) == 6
    done = gen_xyz.xyz_path(xyz_root, 1, 2, 2)
    zero = gen_xyz.xyz_path(xyz_root, 0, 0, 1)
    os.makedirs(os.path.dirname(done))
    os.makedirs(os.path.dirname(zero))
    with open(done, "wb") as f:
        f.write(b"x")
    open(zero, "wb").close()
    scenes, skipped = gen_xyz.plan(sp, xyz_root)
    planned = {i["path"] for s in scenes for _, insts in s[2] for i in insts}
    assert skipped == 1 and len(planned) == 17 and done not in planned and zero in planned
    # the f32 inputs, as the scripts form them
    inst = next(i for s in scenes for _, insts in s[2] for i in insts if i["path"] == zero)
    with open(os.path.join(sp["split_path"], "000000", "scene_gt.json")) as f:
        g = json.load(f)["0"][1]
    assert inst["obj_id"] == g["obj_id"] and inst["t"].dtype == np.float32 and inst["R"].dtype == np.float32
    assert np.array_equal(inst["t"], np.array(g["cam_t_m2c"], dtype="float32") / 1000.0)
    assert np.array_equal(inst["R"], np.array(g["cam_R_m2c"], dtype="float32").reshape(3, 3))


def test_refusals(tmp_path):
    import cv2

    sp, models = _tree(str(tmp_path / "a"))
    os.remove(os.path.join(models, "obj_000002.ply"))
    with pytest.raises(GdrnError, match=r"obj_id 2: no model file .*obj_000002\.ply"):
        gen_xyz.run_split(sp, models)
    sp, models = _tree(str(tmp_path / "b"))
    _edit_json(os.path.join(sp["split_path"], "000001", "scene_camera.json"), lambda c: c.pop("2"))
    with pytest.raises(GdrnError, match="scene 1 image 2: no entry in scene_camera.json"):
        gen_xyz.run_split(sp, models)
    sp, models = _tree(str(tmp_path / "c"))
    os.remove(os.path.join(sp["split_path"], "000001", "rgb", "000002.jpg"))
    with pytest.raises(GdrnError, match=r"missing rgb image .*000001[/\\]rgb[/\\]000002\.jpg"):
        gen_xyz.run_split(sp, models)
    sp, models = _tree(str(tmp_path / "d"))
    cv2.imwrite(os.path.join(sp["split_path"], "000000", "rgb", "000002.jpg"), np.zeros((50, 64, 3), np.uint8))
    with pytest.raises(GdrnError, match=r"image .*000000[/\\]rgb[/\\]000002\.jpg is 64x50, .*000000\.jpg of the same "
                                        r"scene is 64x48"):
        gen_xyz.run_split(sp, models)
    # none of the refusals wrote anything
    assert not os.path.exists(os.path.join(sp["split_path"], "xyz_crop"))


def test_plan_split_default_still_needs_depth(tmp_path):
    sp, _ = _tree(str(tmp_path))
    os.remove(os.path.join(sp["split_path"], "000000", "depth", "000001.png"))
    _edit_json(os.path.join(sp["split_path"], "000001", "scene_camera.json"), lambda c: c["2"].pop("depth_scale"))
    with pytest.raises(GdrnError, match=r"missing depth image .*000000[/\\]depth[/\\]000001\.png"):
        gt_info.plan_split(sp)
    with pytest.raises(GdrnError, match="scene 1 image 2: scene_camera.json has no depth_scale"):
        gt_info.plan_split(sp, [1])
    scenes = gt_info.plan_split(sp, need_depth=False)
    assert [len(ims) for _, ims in scenes] == [3, 3] and "depth" not in scenes[0][1][0]


def _bp_torch_f32(depth, R, t, K):
    """misc.calc_xyz_bp_torch in f32 torch on the CPU (the reference's formula as written)."""
    import torch

    depth, R, T, K = (torch.from_numpy(np.asarray(a, np.float32)) for a in (depth, R, t, K))
    height, width = depth.shape
    mask = (depth != 0).to(depth).view(height, width, 1)
    gy, gx = torch.meshgrid(torch.arange(height, dtype=depth.dtype) - K[1, 2], torch.arange(width, dtype=depth.dtype) - K[0, 2],
                            indexing="ij")
    xyz_cam = torch.stack((gx * depth / K[0, 0], gy * depth / K[1, 1], depth), dim=2).view(height, width, 3, 1)
    Rinv = R.t().view(1, 1, 3, 3).expand(height, width, 3, 3)
    return (torch.einsum("hwij,hwjk->hwi", Rinv, xyz_cam - T.view(1, 1, 3, 1).expand(height, width, 3, 1)) * mask).numpy()


def test_oracle_matches_reference_formula_in_f32():
    rs = np.random.RandomState(0)
    H, W = 60, 80
    K = np.array([[572.4, 0, 41.3], [0, 573.6, 29.7], [0, 0, 1]], np.float32)
    depth = np.zeros((H, W), np.float32)
    depth[11:37, 5:62] = rs.uniform(0.6, 1.4, (26, 57)).astype(np.float32)
    depth[20, 30] = 0
    import cv2

    R = cv2.Rodrigues(rs.uniform(-2, 2, 3))[0].astype(np.float32)
    t = np.array([0.03, -0.02, 1.0], np.float32)
    xyxy, xyz, crop = XO.xyz_crop(depth, R, t, K)
    assert xyxy == [5, 11, 61, 36] and crop.shape == (26, 57, 3) and crop.dtype == np.float16
    ref = _bp_torch_f32(depth, R, t, K)[11:37, 5:62].astype(np.float16)
    d = XO.fp16_ulp_distance(crop, ref)
    assert d.max() <= 1 and (crop[9, 25] == 0).all()
    assert np.array_equal(crop == 0, ref == 0)
    xyxy, _, crop = XO.xyz_crop(np.zeros((H, W), np.float32), R, t, K)
    assert xyxy == [0, 0, W - 1, H - 1] and crop.shape == (H, W, 3) and not crop.any()
    assert XO.fp16_ulp_distance(np.float16([0.0, -0.0, 1.0]), np.float16([-0.0, 2 ** -24, np.nextafter(np.float16(1),
                                                                                                     np.float16(2))])).tolist() == [0, 1, 1]


# ---------------------------------------------------------------------------------------------------------------------
# GPU
def _bop_meshes(n=4, seed=0):
    """Icospheres of ~20k faces (mm), squashed to assorted extents of 60 - 200 mm."""
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    rs = np.random.RandomState(seed)
    return {o: make_icosphere_mesh(5, rs.uniform(60, 200, 3)) for o in range(1, n + 1)}


def _renders(models, obj_index, R, t, K, H, W):
    """The pass's renders: render_meshes of the same f32 poses, near and far."""
    import torch

    from gdrnpp_bop2022_b200 import renderer

    dev = models[0].vertices.device
    n = len(obj_index)
    ids = torch.tensor([models[i].mesh_id for i in obj_index], dtype=torch.int32, device=dev)
    P = np.concatenate([np.asarray(R, np.float32).reshape(n, 3, 3), np.asarray(t, np.float32).reshape(n, 3, 1)], 2)
    return renderer.render_meshes(ids, torch.from_numpy(P).to(dev), torch.from_numpy(np.asarray(K, np.float32)).to(dev),
                                  H, W, gen_xyz.ZNEAR, gen_xyz.ZFAR).cpu().numpy()


def _edge_case_instances(H, W, rs):
    """(obj_index, R, t, K) of instances touching each border, a one-pixel one, one behind the camera, one off-frame
    and a few ordinary ones, at 0.4 - 1.5 m."""
    import cv2

    f = 0.9 * W
    K = np.array([[f, 0, W / 2 - 0.37], [0, f * 1.01, H / 2 + 0.21], [0, 0, 1]], np.float32)
    ts, kinds = [], []
    for k, (u, v) in enumerate([(0, H / 2), (W, H / 3), (W / 3, 0), (W / 2, H), (0, 0)]):   # borders and a corner
        z = 0.5 + 0.25 * k
        ts.append([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z])
        kinds.append("border")
    for z in (0.4, 0.9, 1.5):
        ts.append([rs.uniform(-0.1, 0.1) * z, rs.uniform(-0.1, 0.1) * z, z])
        kinds.append("inside")
    ts.append([0.0, 0.0, -1.0])
    kinds.append("behind")
    ts.append([3.0, 0.0, 1.0])
    kinds.append("off")
    R = np.stack([cv2.Rodrigues(rs.uniform(-2, 2, 3))[0] for _ in ts]).astype(np.float32)
    obj = [k % 4 for k in range(len(ts))]
    return obj, R, np.asarray(ts, np.float32), np.repeat(K[None], len(ts), 0), kinds


def _check_against_oracle(got, depth, R, t, K, H, W, n_diff):
    for i, (xyxy, crop) in enumerate(got):
        rx, _, rc = XO.xyz_crop(depth[i], R[i], t[i], K[i])
        assert xyxy == rx, (i, xyxy, rx)
        assert crop.shape == rc.shape and crop.dtype == np.float16
        assert np.array_equal(crop == 0, rc == 0), i
        d = XO.fp16_ulp_distance(crop, rc)
        assert d.max() <= 1, (i, int(d.max()))
        n_diff[0] += int((d > 0).sum())
        n_diff[1] += d.size


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(480, 640), (960, 1280)])
def test_kernels_match_oracle_on_bop_meshes(lib, dev, H, W):
    from gdrnpp_bop2022_b200 import renderer

    rs = np.random.RandomState(H)
    models = [renderer.Model3D(v * gen_xyz.VERTEX_SCALE, f, device=dev) for v, f in _bop_meshes().values()]
    obj, R, t, K, kinds = _edge_case_instances(H, W, rs)
    # a one-pixel instance: a 0.5 mm sphere whose centre projects onto the centre of pixel (123, 77)
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    tiny = renderer.Model3D(*make_icosphere_mesh(2, (0.0005,) * 3), device=dev)
    models.append(tiny)
    z = 1.2
    K0 = K[0]
    obj.append(len(models) - 1)
    R = np.concatenate([R, np.eye(3, dtype=np.float32)[None]])
    t = np.concatenate([t, np.array([[(123.5 - K0[0, 2]) * z / K0[0, 0], (77.5 - K0[1, 2]) * z / K0[1, 1], z]],
                                    np.float32)])
    K = np.concatenate([K, K0[None]])
    kinds.append("pixel")
    got = gen_xyz.xyz_crops(models, obj, R, t, K, H, W)
    depth = _renders(models, obj, R, t, K, H, W)
    n_diff = [0, 0]
    _check_against_oracle(got, depth, R, t, K, H, W, n_diff)
    boxes = {k: [] for k in set(kinds)}
    for (xyxy, crop), kind in zip(got, kinds):
        boxes[kind].append(xyxy)
    for kind in ("behind", "off"):
        (xyxy,) = boxes[kind]
        crop = got[kinds.index(kind)][1]
        assert xyxy == [0, 0, W - 1, H - 1] and crop.shape == (H, W, 3) and not crop.view(np.uint16).any(), kind
    assert boxes["pixel"] == [[123, 77, 123, 77]] and got[-1][1].shape == (1, 1, 3) and got[-1][1].any()
    b = np.array(boxes["border"])
    assert (b[:, 0] == 0).any() and (b[:, 1] == 0).any() and (b[:, 2] == W - 1).any() and (b[:, 3] == H - 1).any()
    assert all(c.shape[0] > 10 for (_, c), k in zip(got, kinds) if k == "inside")
    print("gen_xyz %dx%d: %d of %d fp16 values differ from fp16(fp64) by 1 ulp" % (W, H, n_diff[0], n_diff[1]))
    # chunking (one instance per chunk, a few, all) and a second call change nothing
    for mb in (1, 3 * gen_xyz.RENDER_BYTES_PER_PIXEL * H * W, 1 << 40):
        again = gen_xyz.xyz_crops(models, obj, R, t, K, H, W, max_bytes=mb)
        assert all(a[0] == g[0] and np.array_equal(a[1].view(np.uint16), g[1].view(np.uint16)) for a, g in zip(again, got))
    assert gen_xyz.xyz_crops(models, [], R[:0], t[:0], K[:0], H, W) == []


@pytest.mark.gpu
def test_pass_renders_equal_egl_renderer_per_instance(lib, dev, tmp_path):
    import torch

    from gdrnpp_bop2022_b200 import renderer
    from gdrnpp_bop2022_b200.ply import save_ply

    H, W = 480, 640
    meshes = _bop_meshes()
    paths = []
    for o, (v, f) in meshes.items():
        paths.append(str(tmp_path / "obj_{:06d}.ply".format(o)))
        save_ply(paths[-1], v, f)
    models = gen_xyz.load_models(str(tmp_path), list(meshes), device=dev)
    model_list = [models[o] for o in sorted(models)]
    egl = renderer.EGLRenderer(paths, vertex_scale=0.001, height=H, width=W, znear=0.01, zfar=6.5, device=dev)
    obj, R, t, K, kinds = _edge_case_instances(H, W, np.random.RandomState(5))
    depth = _renders(model_list, obj, R, t, K, H, W)
    got = gen_xyz.xyz_crops(model_list, obj, R, t, K, H, W)
    seg = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    pc_cam = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    for i in range(len(obj)):
        pose = np.hstack([R[i], t[i].reshape(3, 1)])
        egl.render([obj[i]], [pose], K=K[i], seg_tensor=seg, pc_cam_tensor=pc_cam)
        d = pc_cam[..., 2].cpu().numpy()
        assert np.array_equal(d.view(np.uint32), depth[i].view(np.uint32)), i
        assert np.array_equal((seg[..., 0] > 0).cpu().numpy(), d != 0), i
        # the crop's non-zero pattern is the render's coverage inside the box
        (x1, y1, x2, y2), crop = got[i]
        full = np.zeros((H, W), bool)
        full[y1:y2 + 1, x1:x2 + 1] = crop.any(-1)
        assert np.array_equal(full, d != 0), i


def _split_with_sizes(root):
    """Two scenes of a 640x480 train_pbr split and two of a 720x540 train_primesense split of lmo."""
    from gdrnpp_bop2022_b200.synthetic import write_bop_train_tree

    write_bop_train_tree(root, dataset="lmo", num_images=6, num_scenes=2, insts_per_image=4, num_bg=1)
    write_bop_train_tree(root, dataset="lmo", num_images=4, num_scenes=2, H=540, W=720, insts_per_image=3, num_bg=1,
                         split="train_primesense", seed=1)
    bop = os.path.join(root, "BOP_DATASETS")
    sps = [gt_info.split_params(bop, "lmo", "train", "pbr"), gt_info.split_params(bop, "lmo", "train", "primesense")]
    # an instance behind the camera and one off the frame (every entry gets a file)
    path = os.path.join(sps[0]["split_path"], "000001", "scene_gt.json")

    def edit(c):
        c["2"][0]["cam_t_m2c"] = [0.0, 0.0, -800.0]
        c["2"][2]["cam_t_m2c"] = [5000.0, 0.0, 800.0]
    _edit_json(path, edit)
    return bop, sps


def _read_files(xyz_root):
    out = {}
    for d in sorted(os.listdir(xyz_root)):
        for name in sorted(os.listdir(os.path.join(xyz_root, d))):
            with open(os.path.join(xyz_root, d, name), "rb") as f:
                out[(d, name)] = f.read()
    return out


@pytest.mark.gpu
def test_split_end_to_end_against_oracle_files(lib, dev, tmp_path):
    import torch

    root = str(tmp_path / "datasets")
    bop, sps = _split_with_sizes(root)
    model_dir = gt_info.models_path(bop, "lmo")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "gdrnpp_bop2022_b200.gen_xyz", "--dataset", "lmo", "--dataset_split",
                        "train", "--dataset_split_type", "pbr", "--datasets_path", bop], check=True, cwd=str(tmp_path),
                       env=env, capture_output=True, text=True)
    totals = json.loads(r.stdout.strip().splitlines()[-1])
    assert totals["images"] == 6 and totals["written"] == 24 and totals["skipped"] == 0 and totals["empty"] == 2
    assert "not visible: scene 1 image 2 entry 0 obj_id" in r.stdout and "entry 2 obj_id" in r.stdout
    r2 = gen_xyz.run_split(sps[1], model_dir, device=dev, log=None)
    assert r2["written"] == 12 and r2["empty"] == 0
    models = gen_xyz.load_models(model_dir, [1, 2, 3], device=dev)
    order = sorted(models)
    n_equal = n_files = 0
    for sp, (H, W) in zip(sps, [(480, 640), (540, 720)]):
        xyz_root = os.path.join(sp["split_path"], "xyz_crop")
        files = _read_files(xyz_root)
        n_entries = 0
        for scene_id, ims in gt_info.plan_split(sp, need_depth=False):
            for im in ims:
                gts = im["gts"]
                n_entries += len(gts)
                R = np.stack([np.asarray(g["cam_R_m2c"], np.float32).reshape(3, 3) for g in gts])
                t = np.stack([np.asarray(g["cam_t_m2c"], np.float32).reshape(3) / np.float32(1000.0) for g in gts])
                K = np.repeat(np.asarray(im["K"], np.float32).reshape(1, 3, 3), len(gts), 0)
                obj = [order.index(int(g["obj_id"])) for g in gts]
                depth = _renders([models[o] for o in order], obj, R, t, K, H, W)
                for j in range(len(gts)):
                    raw = files[("{:06d}".format(scene_id), "{:06d}_{:06d}-xyz.pkl".format(im["im_id"], j))]
                    got = pickle.loads(raw)
                    assert list(got) == ["xyz_crop", "xyxy"] and all(type(v) is int for v in got["xyxy"])
                    ref = XO.file_dict(depth[j], R[j], t[j], K[j])
                    assert got["xyxy"] == ref["xyxy"] and got["xyz_crop"].dtype == np.float16
                    assert XO.fp16_ulp_distance(got["xyz_crop"], ref["xyz_crop"]).max() <= 1
                    assert raw == pickle.dumps({"xyz_crop": got["xyz_crop"], "xyxy": ref["xyxy"]}, protocol=2)
                    if np.array_equal(got["xyz_crop"].view(np.uint16), ref["xyz_crop"].view(np.uint16)):
                        assert raw == pickle.dumps(ref, protocol=2)
                        n_equal += 1
                    n_files += 1
                    # data_loader.py: paste the crop into the frame, mask_obj = any component != 0
                    x1, y1, x2, y2 = got["xyxy"]
                    xyz = np.zeros((H, W, 3), dtype=np.float32)
                    xyz[y1:y2 + 1, x1:x2 + 1, :] = got["xyz_crop"]
                    mask_obj = ((xyz[:, :, 0] != 0) | (xyz[:, :, 1] != 0) | (xyz[:, :, 2] != 0)).astype(np.float32)
                    assert np.array_equal(mask_obj, (depth[j] != 0).astype(np.float32))
        assert len(files) == n_entries
    assert n_files == 36 and n_equal > 0
    print("gen_xyz end to end: %d of %d files byte-equal to the oracle's" % (n_equal, n_files))
    # resume: a planted non-empty file keeps its bytes and mtime, a planted empty file is rewritten
    xyz_root = os.path.join(sps[0]["split_path"], "xyz_crop")
    before = _read_files(xyz_root)
    keep = os.path.join(xyz_root, "000000", "000001_000002-xyz.pkl")
    redo = os.path.join(xyz_root, "000001", "000002_000001-xyz.pkl")
    with open(keep, "wb") as f:
        f.write(b"planted")
    os.utime(keep, ns=(1_000_000_000, 1_000_000_000))
    open(redo, "wb").close()
    r3 = gen_xyz.run_split(sps[0], model_dir, device=dev, log=None)
    assert r3["written"] == 1 and r3["skipped"] == 23
    after = _read_files(xyz_root)
    assert after[("000000", "000001_000002-xyz.pkl")] == b"planted" and os.stat(keep).st_mtime_ns == 1_000_000_000
    assert after[("000001", "000002_000001-xyz.pkl")] == before[("000001", "000002_000001-xyz.pkl")]
    assert not any(name.endswith(".tmp") for _, name in after)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_driver_files_identical_across_chunking_and_runs(lib, dev, tmp_path):
    root = str(tmp_path / "datasets")
    bop, sps = _split_with_sizes(root)
    model_dir = gt_info.models_path(bop, "lmo")
    runs = []
    for kw in ({"max_bytes": 1}, {"max_bytes": 1 << 40, "batch_images": 100}, {"batch_images": 1}, {}):
        for sp in sps:
            shutil.rmtree(os.path.join(sp["split_path"], "xyz_crop"), ignore_errors=True)
            r = gen_xyz.run_split(sp, model_dir, device=dev, log=None, **kw)
            assert r["skipped"] == 0
        runs.append([_read_files(os.path.join(sp["split_path"], "xyz_crop")) for sp in sps])
    for o in runs[1:]:
        assert o == runs[0]
    assert len(runs[0][0]) == 24 and len(runs[0][1]) == 12
