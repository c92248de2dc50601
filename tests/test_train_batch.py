"""GPU training batches (gdrnpp_bop2022_b200/train_batch.py, csrc/train_aug.cu) against the NumPy / cv2 / PIL
restatement of read_data_train (oracle/train_batch_oracle.py)."""
import copy
import json
import os
import pickle
import shutil

import numpy as np
import pytest

from gdrnpp_bop2022_b200 import train_batch as TB

# the COLOR_AUG_CODE every shipped GDRN config uses (configs/gdrn/*/convnext_AugCosyAAEGray_*)
SHIPPED_CODE = (
    "Sequential(["
    "Sometimes(0.5, CoarseDropout( p=0.2, size_percent=0.05) ),"
    "Sometimes(0.4, GaussianBlur((0., 3.))),"
    "Sometimes(0.3, pillike.EnhanceSharpness(factor=(0., 50.))),"
    "Sometimes(0.3, pillike.EnhanceContrast(factor=(0.2, 50.))),"
    "Sometimes(0.5, pillike.EnhanceBrightness(factor=(0.1, 6.))),"
    "Sometimes(0.3, pillike.EnhanceColor(factor=(0., 20.))),"
    "Sometimes(0.5, Add((-25, 25), per_channel=0.3)),"
    "Sometimes(0.3, Invert(0.2, per_channel=True)),"
    "Sometimes(0.5, Multiply((0.6, 1.4), per_channel=0.5)),"
    "Sometimes(0.5, Multiply((0.6, 1.4))),"
    "Sometimes(0.1, AdditiveGaussianNoise(scale=10, per_channel=True)),"
    "Sometimes(0.5, iaa.contrast.LinearContrast((0.5, 2.2), per_channel=0.3)),"
    "Sometimes(0.5, Grayscale(alpha=(0.0, 1.0))),"
    "], random_order=True)"
)


def shipped_cfg(train=("ycbv_train_pbr",)):
    from gdrnpp_bop2022_b200.synthetic import shipped_train_cfg

    return shipped_train_cfg(train)


def test_synthetic_config_carries_the_shipped_program():
    from gdrnpp_bop2022_b200.synthetic import SHIPPED_COLOR_AUG_CODE

    assert SHIPPED_COLOR_AUG_CODE == SHIPPED_CODE


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    from gdrnpp_bop2022_b200.synthetic import write_bop_train_tree

    root = str(tmp_path_factory.mktemp("train"))
    base = write_bop_train_tree(root, num_images=8, num_scenes=2, insts_per_image=4, seed=3)
    return root, base


def _write_fps(base):
    """fps_points.pkl without the native library: the eight box corners (any points do for the host tests)."""
    from gdrnpp_bop2022_b200.ply import load_ply

    out = {}
    for o in (1, 2, 3):
        pts = load_ply(os.path.join(base, "models", "obj_{:06d}.ply".format(o)), vertex_scale=0.001)["pts"]
        out[str(o)] = {f"fps{n}_and_center": np.concatenate([pts[np.arange(n) % len(pts)], pts.mean(0, keepdims=True)])
                       for n in TB.FPS_COUNTS}
    with open(os.path.join(base, "models", "fps_points.pkl"), "wb") as f:
        pickle.dump(out, f)


# ------------------------------------------------------------------------------------------------ CPU
def test_trainset_filters_and_per_object_fields(tree):
    root, base = tree
    fps_path = os.path.join(base, "models", "fps_points.pkl")
    if os.path.exists(fps_path):
        os.remove(fps_path)
    cfg = shipped_cfg()
    with pytest.raises(TB.GdrnError, match="compute_fps"):
        TB.TrainSet(cfg, root)
    _write_fps(base)
    ts = TB.TrainSet(cfg, root)
    expect = 0
    for s in ("000000", "000001"):
        info = json.load(open(os.path.join(base, "train_pbr", s, "scene_gt_info.json")))
        for im in info.values():
            expect += sum(g["bbox_visib"][2] > 1 and g["bbox_visib"][3] > 1 and g["px_count_visib"] > 0
                          and g["visib_fract"] > 0.3 for g in im)
    assert len(ts) == expect and 0 < expect < 32
    assert ts.obj_ids == [1, 2, 3]
    assert ts.roi_points.shape == (3, 8, 3) and ts.extents.shape == (3, 3) and ts.fps_points.shape == (3, 64, 3)
    assert ts.sym_info[0] is None and ts.sym_info[1].shape == (2, 3, 3) and ts.sym_info[2] is None
    s = ts.samples[0]
    assert set(s) >= {"rgb", "mask_visib", "mask", "K", "R", "t", "label", "bbox_obj", "bbox_visib", "centroid"}
    one = TB.TrainSet(shipped_cfg(("ycbv_003_cracker_box_train_pbr",)), root)
    assert one.obj_ids == [2] and all(x["label"] == 0 for x in one.samples)
    with pytest.raises(TB.GdrnError, match="not a supported BOP train split"):
        TB.TrainSet(shipped_cfg(("lmo_train_real",)), root)


def test_color_aug_parser():
    ops, random_order = TB.parse_color_aug(SHIPPED_CODE)
    assert random_order and [o["kind"] for o in ops] == [
        "CoarseDropout", "GaussianBlur", "EnhanceSharpness", "EnhanceContrast", "EnhanceBrightness", "EnhanceColor", "Add",
        "Invert", "Multiply", "Multiply", "AdditiveGaussianNoise", "LinearContrast", "Grayscale"]
    assert [o["prob"] for o in ops] == [0.5, 0.4, 0.3, 0.3, 0.5, 0.3, 0.5, 0.3, 0.5, 0.5, 0.1, 0.5, 0.5]
    assert ops[6]["value"] == (-25, 25) and ops[6]["per_channel"] == 0.3 and ops[0]["size_percent"] == 0.05
    with pytest.raises(TB.GdrnError, match="'Superpixels' is not supported"):
        TB.parse_color_aug("Sequential([Sometimes(0.5, Superpixels(0.5))])")
    with pytest.raises(TB.GdrnError, match="not a literal"):
        TB.parse_color_aug("Sequential([GaussianBlur(1.2*np.random.rand())])")


@pytest.mark.parametrize("key,value,msg", [
    ("INPUT.WITH_DEPTH", True, "INPUT.WITH_DEPTH"),
    ("INPUT.MIN_SIZE_TRAIN", (400,), "INPUT.MIN_SIZE_TRAIN"),
    ("INPUT.DZI_TYPE", "roi10d", "INPUT.DZI_TYPE"),
    ("MODEL.POSE_NET.XYZ_ONLINE", False, "XYZ_ONLINE"),
    ("MODEL.POSE_NET.LOSS_CFG.XYZ_LOSS_TYPE", "CE_coor", "XYZ_LOSS_TYPE"),
    ("MODEL.POSE_NET.PNP_NET.COORD_2D_TYPE", "rel", "COORD_2D_TYPE"),
    ("TRAIN.VIS", True, "TRAIN.VIS"),
    ("INPUT.BG_TYPE", "SUN_RGBD", "SUN_RGBD"),
    ("INPUT.COLOR_AUG_TYPE", "ROI10D", "COLOR_AUG_TYPE"),
])
def test_rejected_settings(key, value, msg):
    cfg = copy.deepcopy(shipped_cfg())
    TB.check_train_config(cfg, (480, 640))
    d = cfg
    *path, last = key.split(".")
    for p in path:
        d = d[p]
    d[last] = value
    with pytest.raises(NotImplementedError, match=msg):
        TB.check_train_config(cfg, (480, 640))


def test_train_resize_must_be_the_identity_for_the_split(tmp_path):
    from gdrnpp_bop2022_b200.synthetic import write_bop_train_tree

    root = str(tmp_path)
    base = write_bop_train_tree(root, dataset="tless", num_images=2, num_scenes=1, H=540, W=720, insts_per_image=2,
                                seed=5, num_bg=1)
    _write_fps(base)
    shutil.copytree(os.path.join(base, "models"), os.path.join(base, "models_cad"))   # T-LESS trains on the CAD models
    cfg = shipped_cfg(("tless_1_train_pbr",))
    # the default 480 / 640 resizes T-LESS's 720x540 images: refused before any device work
    with pytest.raises(NotImplementedError, match="resize the 720x540 training images"):
        TB.GdrnTrainBatcher(cfg, root, device="cpu")
    # configs/gdrn/tlessPbrSO: 540 / 720, the identity for these images
    cfg["INPUT"].update(MIN_SIZE_TRAIN=(540,), MAX_SIZE_TRAIN=720)
    TB.check_train_config(cfg, (540, 720))
    with pytest.raises(NotImplementedError, match="MIN_SIZE_TRAIN"):
        TB.check_train_config(cfg, (480, 640))
    # configs/gdrn/itoddPbrSO: 960 / 1280 on ITODD's 1280x960 images; a "range" must hold for every length in it
    cfg["INPUT"].update(MIN_SIZE_TRAIN=(960,), MAX_SIZE_TRAIN=1280)
    TB.check_train_config(cfg, (960, 1280))
    cfg["INPUT"].update(MIN_SIZE_TRAIN=(950, 960), MIN_SIZE_TRAIN_SAMPLING="range")
    with pytest.raises(NotImplementedError, match="shortest edge 950"):
        TB.check_train_config(cfg, (960, 1280))
    cfg["INPUT"].update(IMG_AUG_RESIZE=False)
    TB.check_train_config(cfg, (960, 1280))


@pytest.mark.parametrize("code,msg", [
    ("Sequential([GaussianBlur((0., 5.))])", "15-tap kernel"),
    ("Sequential([GaussianBlur(4.2)])", "13-tap kernel"),
    ("Sequential([CoarseDropout(0.1, size_percent=(0.02, 0.05))])", "only a fixed size_percent"),
    ("Sequential([CoarseDropout(0.1, size_percent=0.05), CoarseDropout(0.2, size_percent=0.05)])", "at most one"),
    ("Sequential([Add([-10, 10])])", "lists"),
    ("Sequential([Multiply((0.5, 1.0, 2.0))])", "a range must be a pair of numbers"),
])
def test_parser_rejects_what_the_records_cannot_hold(code, msg):
    with pytest.raises(TB.GdrnError, match=msg):
        TB.parse_color_aug(code)


def test_parser_accepts_ranges_the_sampler_draws():
    code = ("Sequential([CoarseDropout((0.02, 0.1), size_percent=0.05), GaussianBlur((0., 4.1)), Invert((0.1, 0.3)),"
            "Add(7)])")
    ops, _ = TB.parse_color_aug(code)
    cfg = shipped_cfg()
    cfg["INPUT"]["COLOR_AUG_CODE"] = code
    sm = TB.Sampler(cfg, 10, 1, (480, 640))
    r = sm.draw(np.random.default_rng(0), 200)
    on = r["do_color"] > 0
    drop = 1 - r["cells"][on].reshape(on.sum(), -1).mean(1)
    assert 0.0 < drop.min() and drop.max() < 0.2
    blur = r["kind_at"] == TB.COLOR_OPS["GaussianBlur"]
    assert blur.any() and r["ipar"][blur][:, 0].max() <= TB.MAX_BLUR_TAPS
    assert (r["ipar"][r["kind_at"] == TB.COLOR_OPS["Add"]][:, :3] == 7).all()


@pytest.mark.parametrize("bbox_type,dzi", [("AMODAL_CLIP", "uniform"), ("VISIB", "uniform"), ("AMODAL_CLIP", "none")])
def test_roi_geometry_equals_the_reference_formulas(tree, bbox_type, dzi):
    from oracle import train_batch_oracle as O

    root, base = tree
    _write_fps(base)
    cfg = shipped_cfg()
    cfg["MODEL"]["BBOX_TYPE"] = bbox_type
    cfg["INPUT"]["DZI_TYPE"] = dzi
    ts = TB.TrainSet(cfg, root)
    ts.im_size = (480, 640)
    rec = TB.Sampler(cfg, len(ts), 1, ts.im_size).draw(np.random.default_rng(8), 64)
    ours, ref = TB.roi_geometry(cfg, ts, rec), O.roi_geometry(cfg, ts, rec)
    clipped = sum(s["bbox_obj"][0] < 0 or s["bbox_obj"][0] + s["bbox_obj"][2] > 640 for s in ts.samples)
    assert clipped > 0   # the split has boxes that AMODAL_CLIP clips
    for k in ("center", "scale", "wh", "trans_ratio"):
        np.testing.assert_allclose(ours[k], ref[k], rtol=1e-12, atol=1e-12, err_msg=k)


def test_gaussian_kernel_reproduces_cv2():
    import cv2

    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (60, 80, 3), dtype=np.uint8)
    for sigma in [0.0011, 0.01, 0.3, 0.5, 1.0, 2.0, 2.999] + list(rng.uniform(0, 3, 40)):
        sigma = float(np.float32(sigma))
        n = TB.gaussian_ksize(sigma)
        k = TB.gaussian_kernel_u8(sigma, n).astype(np.int64)
        assert k.sum() == 256
        r = n // 2
        p = np.pad(img.astype(np.int64), ((r, r), (r, r), (0, 0)), mode="reflect")
        h = sum(k[j] * p[:, j:j + 80] for j in range(n))
        v = sum(k[j] * h[j:j + 60] for j in range(n))
        ours = np.clip((v + 32768) >> 16, 0, 255).astype(np.uint8)
        ref = cv2.GaussianBlur(img, (n, n), sigmaX=sigma, sigmaY=sigma, borderType=cv2.BORDER_REFLECT_101)
        assert np.array_equal(ours, ref), sigma


def test_pillike_oracle_equals_pil():
    from PIL import Image, ImageEnhance

    from oracle import train_batch_oracle as O

    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    P = Image.fromarray(img)
    for kind in ("Sharpness", "Contrast", "Brightness", "Color"):
        for f in (0.0, 0.1, 0.2, 0.5, 1.0, 1.7, 6.0, 20.0, 50.0):
            ref = np.asarray(getattr(ImageEnhance, kind)(P).enhance(float(np.float32(f))))
            assert np.array_equal(O.enhance(img, "Enhance" + kind, np.float32(f)), ref), (kind, f)


def test_grayscale_oracle_uses_cv2_luma():
    import cv2

    from oracle import train_batch_oracle as O

    img = np.random.default_rng(2).integers(0, 256, (480, 640, 3), dtype=np.uint8)
    g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
    assert np.array_equal(O.grayscale(img, 1.0), np.repeat(g[..., None], 3, 2))


def test_records_deterministic_and_frequencies():
    cfg = shipped_cfg()
    sm = TB.Sampler(cfg, 1000, 50, (480, 640))
    a = sm.draw(np.random.default_rng([5, 1]), 64)
    b = sm.draw(np.random.default_rng([5, 1]), 64)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    n = 100_000
    # the cell grid is what costs memory: draw the big sample with a 1x1 grid
    sm.cell_hw = (1, 1)
    r = sm.draw(np.random.default_rng(7), n)

    def within(count, total, p):
        return abs(count - total * p) <= 5 * np.sqrt(total * p * (1 - p)) + 1

    assert within(r["do_bg"].sum(), n, 0.5)
    assert within(r["do_color"].sum(), n, 0.8)
    col = r["do_color"] > 0
    for c, op in enumerate(sm.ops):
        assert within(r["op_on"][col, c].sum(), col.sum(), op["prob"]), op["kind"]
    sides = r["trunc_side"][r["do_bg"] > 0]
    for s in range(5):
        assert within((sides == s).sum(), sides.size, 0.2)
    # every op lands at every position with probability 1/13
    perm = r["perm"][col]
    for c in range(13):
        hist = np.bincount(np.nonzero(perm == c)[1], minlength=13)
        assert all(within(h, perm.shape[0], 1 / 13) for h in hist)
    assert np.all(np.abs(r["dzi_scale"] - 1) <= 0.25) and np.all(np.abs(r["dzi_shift"]) <= 0.25)


def test_bg_layout_matches_get_bg_image():
    # 640x480 image: a 500x375 background keeps its aspect (no crop), a portrait one is cropped to the image's aspect
    assert TB.bg_layout((375, 500), 480, 640)[:4] == (375, 500, 480, 640)
    ch, cw, rh, rw, _ = TB.bg_layout((500, 375), 480, 640)
    assert (ch, cw) == (282, 375) and rh <= 480 and rw <= 640


# ------------------------------------------------------------------------------------------------ GPU
def _rand_images(n, seed, H=480, W=640):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


def _run_step(dev, imgs, kind, fpar, ipar, cells):
    import torch

    from gdrnpp_bop2022_b200 import _lib

    n, H, W, _ = imgs.shape
    L = _lib.lib()
    src = torch.from_numpy(imgs).to(dev)
    dst = torch.empty_like(src)
    kind_d = torch.tensor(np.asarray(kind, np.int32).reshape(n, 1), device=dev)
    fp = torch.from_numpy(np.asarray(fpar, np.float32).reshape(n, 1, 4)).to(dev)
    ip = torch.from_numpy(np.asarray(ipar, np.int32).reshape(n, 1, 12)).to(dev)
    ce = torch.from_numpy(np.ascontiguousarray(cells, np.uint8)).to(dev)
    sums = torch.zeros(n, dtype=torch.int64, device=dev)
    _lib.check(L.gdrn_train_luma_sum(_lib.ptr(src), n, H, W, _lib.ptr(kind_d), 1, 0, _lib.ptr(sums), _lib.current_stream()),
               "luma")
    _lib.check(L.gdrn_train_color_step(_lib.ptr(src), _lib.ptr(dst), n, H, W, _lib.ptr(kind_d), _lib.ptr(fp), _lib.ptr(ip), 1,
                                       0, _lib.ptr(ce), cells.shape[1], cells.shape[2], _lib.ptr(sums),
                                       _lib.current_stream()), "step")
    return dst.cpu().numpy()


def _op_cases():
    rng = np.random.default_rng(11)
    K = TB.COLOR_OPS
    cases = []
    for sigma in (0.0, 0.0009, 0.3, 1.0, 2.2, 2.9999):
        i = np.zeros(12, np.int32)
        if sigma > TB.BLUR_EPS:
            k = TB.gaussian_ksize(sigma)
            i[0] = k
            i[1:1 + k] = TB.gaussian_kernel_u8(float(np.float32(sigma)), k)
        cases.append(("GaussianBlur", K["GaussianBlur"] if sigma > TB.BLUR_EPS else -1, [sigma, 0, 0, 0], i))
    for name, lo, hi in (("EnhanceSharpness", 0.0, 50.0), ("EnhanceContrast", 0.2, 50.0), ("EnhanceBrightness", 0.1, 6.0),
                         ("EnhanceColor", 0.0, 20.0)):
        for f in (lo, hi, 1.0, rng.uniform(lo, hi)):
            cases.append((name, K[name], [f, 0, 0, 0], np.zeros(12, np.int32)))
    for v in ((-25, -25, -25), (25, 25, 25), (3, -7, 19)):
        cases.append(("Add", K["Add"], [0] * 4, np.array(list(v) + [0] * 9, np.int32)))
    for fl in ((1, 0, 1), (0, 0, 0), (1, 1, 1)):
        cases.append(("Invert", K["Invert"], [0] * 4, np.array(list(fl) + [0] * 9, np.int32)))
    for m in ((0.6, 0.6, 0.6), (1.4, 1.4, 1.4), (0.77, 1.21, 1.03)):
        cases.append(("Multiply", K["Multiply"], list(m) + [0], np.zeros(12, np.int32)))
    for a in ((0.5, 0.5, 0.5), (2.2, 2.2, 2.2), (0.8, 1.6, 2.0)):
        cases.append(("LinearContrast", K["LinearContrast"], list(a) + [0], np.zeros(12, np.int32)))
    for a in (0.0, 1.0, 0.37):
        cases.append(("Grayscale", K["Grayscale"], [a, 0, 0, 0], np.zeros(12, np.int32)))
    for seed in ((1, 2), (123456789, -5)):
        cases.append(("AdditiveGaussianNoise", K["AdditiveGaussianNoise"], [10.0, 0, 0, 0],
                      np.array(list(seed) + [0] * 10, np.int32)))
    cases.append(("CoarseDropout", K["CoarseDropout"], [0] * 4, np.zeros(12, np.int32)))
    return cases


@pytest.mark.gpu
def test_color_ops_equal_oracle(lib, dev):
    from PIL import Image, ImageEnhance

    from oracle import train_batch_oracle as O

    cases = _op_cases()
    n = len(cases)
    imgs = _rand_images(n, 0)
    imgs[: n // 2] = np.stack([np.asarray(Image.fromarray(im).resize((640, 480))) for im in
                               _rand_images(n // 2, 1, 120, 160)])   # smooth ones too, so blends land between levels
    cells = (np.random.default_rng(2).random((n, 24, 32)) >= 0.2).astype(np.uint8)
    kind = [c[1] for c in cases]
    fpar = np.array([np.float32(c[2]) for c in cases], np.float32)
    ipar = np.stack([c[3] for c in cases])
    got = _run_step(dev, imgs, kind, fpar, ipar, cells)
    for b, (name, k, _, _) in enumerate(cases):
        ref = O.apply_op(imgs[b], k, fpar[b], ipar[b], cells[b])
        assert np.array_equal(got[b], ref), (name, fpar[b], ipar[b][:3], int((got[b] != ref).sum()))
        if name.startswith("Enhance"):
            pil = getattr(ImageEnhance, name[len("Enhance"):])(Image.fromarray(imgs[b])).enhance(float(fpar[b][0]))
            assert np.array_equal(got[b], np.asarray(pil)), name


def _batcher(tree, dev, **kw):
    root, base = tree
    if not os.path.exists(os.path.join(base, "models", "fps_points.pkl")):
        _write_fps(base)
    cfg = shipped_cfg()
    cfg["INPUT"].update(kw.pop("input", {}))
    return TB.GdrnTrainBatcher(cfg, root, device=dev, **kw)


@pytest.mark.gpu
def test_background_composite_all_sides(lib, dev, tree):
    import torch

    from oracle import train_batch_oracle as O

    bt = _batcher(tree, dev, seed=1, batch_size=20, num_workers=2, input={"COLOR_AUG_PROB": 0.0, "CHANGE_BG_PROB": 1.0})
    rec = bt.sampler.draw(np.random.default_rng(3), 20)
    rec["trunc_side"][:] = np.arange(20) % 5   # every side, and no truncation
    rec["bg_index"][:] = np.arange(20) % len(bt.bg_paths)
    with torch.cuda.device(dev):
        out = TB.build_images(bt.cfg, bt.ts, rec, TB.decode(bt.ts, bt.bg_paths, rec), dev)
    ref = O.replay(bt.cfg, bt.ts, bt.bg_paths, rec)
    assert np.array_equal(out["image"].cpu().numpy(), ref["image"])
    for key in ("roi_mask_trunc", "roi_mask_visib", "roi_mask_full", "roi_img", "roi_coord_2d"):
        assert np.array_equal(out[key].cpu().numpy(), ref[key]), key
    assert np.array_equal(out["counts"].cpu().numpy(), ref["counts"])
    bt.close()


@pytest.mark.gpu
def test_whole_batch_equals_oracle_and_targets(lib, dev, tree):
    import torch

    from gdrnpp_bop2022_b200.online_targets import render_roi_targets
    from oracle import train_batch_oracle as O

    bt = _batcher(tree, dev, seed=4, batch_size=48, num_workers=4)
    batch = next(bt)
    rec = bt.last_records
    ref = O.replay(bt.cfg, bt.ts, bt.bg_paths, rec)
    assert (rec["do_color"] > 0).any() and (rec["do_bg"] > 0).any()
    assert np.array_equal(bt.last_images.cpu().numpy(), ref["image"])
    for key in ("roi_img", "roi_coord_2d"):
        assert np.array_equal(batch[key].cpu().numpy(), ref[key]), key
    tg = render_roi_targets(bt.models, batch["roi_cls"], batch["ego_rot"], batch["trans"], batch["roi_zoom_K"],
                            batch["roi_extent"], batch["roi_fps_points"], out_res=64)
    obj = tg["roi_mask_obj"].cpu().numpy()
    assert obj.sum() > 0
    for key in ("roi_xyz", "roi_region", "roi_mask_obj"):
        assert torch.equal(batch[key], tg[key]), key
    assert np.array_equal(batch["roi_mask_trunc"].cpu().numpy(), ref["roi_mask_trunc"] * obj)
    assert np.array_equal(batch["roi_mask_visib"].cpu().numpy(), ref["roi_mask_visib"] * obj)
    assert np.array_equal(batch["roi_mask_full"].cpu().numpy(), ref["roi_mask_full"])
    assert (ref["counts"] >= 32).all()
    # the scalar keys against the oracle's restatement of the reference's box arithmetic
    geo = O.roi_geometry(bt.cfg, bt.ts, rec)
    samples = [bt.ts.samples[i] for i in rec["index"]]
    np.testing.assert_allclose(batch["roi_center"].cpu().numpy(), geo["center"], rtol=1e-6, atol=1e-4)
    np.testing.assert_allclose(batch["roi_scale"].cpu().numpy(), geo["scale"], rtol=1e-6)
    np.testing.assert_allclose(batch["resize_ratio"].cpu().numpy(), 64 / geo["scale"], rtol=1e-6)
    np.testing.assert_allclose(batch["roi_trans_ratio"].cpu().numpy(), geo["trans_ratio"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(batch["roi_wh"].cpu().numpy(), geo["wh"], rtol=1e-6)
    K = np.stack([s["K"] for s in samples]).astype(np.float64)
    crop = geo["center"].astype(np.float32).astype(np.float64) - geo["scale"].astype(np.float32)[:, None] / 2
    Kz = K.copy()
    Kz[:, :2, 2] -= crop
    Kz[:, :2] *= (64 / geo["scale"].astype(np.float32).astype(np.float64))[:, None, None]
    np.testing.assert_allclose(batch["roi_zoom_K"].cpu().numpy(), Kz, rtol=1e-6, atol=1e-4)
    assert batch["roi_cls"].dtype == torch.long and batch["roi_region"].dtype == torch.long
    assert batch["roi_img"].shape == (48, 3, 256, 256) and batch["roi_xyz"].shape == (48, 3, 64, 64)
    assert batch["roi_points"].shape == (48, 8, 3) and isinstance(batch["sym_info"], list) and len(batch["sym_info"]) == 48
    assert set(batch) == {"roi_img", "roi_cls", "roi_coord_2d", "roi_cam", "roi_center", "roi_scale", "resize_ratio",
                          "roi_zoom_K", "roi_wh", "roi_extent", "roi_trans_ratio", "roi_mask_trunc", "roi_mask_visib",
                          "roi_mask_full", "ego_rot", "trans", "roi_points", "sym_info", "roi_mask_obj",
                          "roi_fps_points", "roi_region", "roi_xyz"}
    # same seed, same batches
    bt2 = _batcher(tree, dev, seed=4, batch_size=48, num_workers=2)
    again = next(bt2)
    for key, v in batch.items():
        if torch.is_tensor(v):
            assert torch.equal(v, again[key]), key
    bt.close()
    bt2.close()


@pytest.mark.gpu
def test_redraw_replaces_small_masks(lib, dev, tree):
    bt = _batcher(tree, dev, seed=9, batch_size=16, num_workers=2)
    tiny = dict(bt.ts.samples[0])
    tiny["bbox_obj"] = tiny["bbox_visib"] = [0, 0, 2, 2]   # a ~3-pixel crop of the image corner: < 32 mask pixels
    bt.ts.samples.append(tiny)
    tiny_idx = len(bt.ts.samples) - 1
    orig, calls = bt.sampler.draw, []

    def draw(rng, n):
        r = orig(rng, n)
        if not calls:
            r["index"][0] = tiny_idx
        calls.append(n)
        return r

    bt.sampler.draw = draw
    batch = next(bt)
    # draws: this batch, the prefetched next one, then the redraw of the rejected slot(s)
    assert len(calls) >= 3 and calls[0] == 16 and calls[2] >= 1
    assert bt.last_records["index"][0] != tiny_idx
    from oracle import train_batch_oracle as O

    ref = O.replay(bt.cfg, bt.ts, bt.bg_paths, bt.last_records)
    assert (ref["counts"] >= 32).all()
    assert np.array_equal(batch["roi_img"].cpu().numpy(), ref["roi_img"])
    bt.close()


@pytest.mark.gpu
def test_compute_fps_matches_native(lib, dev, tmp_path):
    from gdrnpp_bop2022_b200.native_ops import farthest_point_sampling
    from gdrnpp_bop2022_b200.ply import load_ply, save_ply
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    v, f = make_icosphere_mesh(3, (120.0, 80.0, 60.0))
    models = tmp_path / "BOP_DATASETS" / "ycbv" / "models"
    os.makedirs(models)
    save_ply(str(models / "obj_000001.ply"), v, f)
    (models / "models_info.json").write_text(json.dumps({"1": {"diameter": 120.0}}))
    TB.main(["compute_fps", "--dataset", "ycbv", "--datasets-root", str(tmp_path)])
    res = pickle.load(open(models / "fps_points.pkl", "rb"))
    pts = load_ply(str(models / "obj_000001.ply"), vertex_scale=0.001)["pts"].astype(np.float32)
    for n in TB.FPS_COUNTS:
        e = res["1"][f"fps{n}_and_center"]
        assert e.shape == (n + 1, 3)
        assert np.array_equal(e[:-1], farthest_point_sampling(pts, n, init_center=True))
        np.testing.assert_array_equal(e[-1], [np.average(pts[:, i]) for i in range(3)])   # get_fps_and_center
