"""The dataset test loop (gdrn_evaluator.py, main_gdrn.py) and its batched ROI-input kernels (csrc/roi_batch.cu)."""
import json
import os
import types

import numpy as np
import pytest
import torch

from gdrnpp_bop2022_b200 import gdrn_evaluator as G
from gdrnpp_bop2022_b200.gdrn_model import default_cfg


def _cfg(det_file="datasets/none.json", dataset="ycbv", **test):
    cfg = default_cfg(with_maps=False)
    cfg.VAL = types.SimpleNamespace(DATASET_NAME=dataset, SPLIT="test", SPLIT_TYPE="", TARGETS_FILENAME="test_targets_bop19.json",
                                    USE_BOP=True, EVAL_CACHED=False, SAVE_BOP_CSV_ONLY=False, ERROR_TYPES="ad,reteS,proj",
                                    N_TOP=-1, SCORE_ONLY=False, RENDERER_TYPE="cpp")
    cfg.DATASETS = types.SimpleNamespace(DET_FILES_TEST=(det_file,), DET_THR=0.0, DET_TOPK_PER_OBJ=100)
    cfg.INPUT = types.SimpleNamespace(WITH_DEPTH=False, DZI_PAD_SCALE=1.5, MIN_SIZE_TEST=480, MAX_SIZE_TEST=640)
    for k, v in test.items():
        setattr(cfg.TEST, k, v)
    return cfg


# ---------------------------------------------------------------------------------------------------- CPU
def _ref_load_detections(detections, scene_im_ids, objs, id2obj, score_thr, top_k_per_obj, train_objs):
    """load_detections_into_dataset (core/utils/dataset_utils.py:146-235), restated on names as the reference does."""
    out = []
    for scene_im_id in scene_im_ids:
        if scene_im_id not in detections:
            continue
        obj_annotations = {obj: [] for obj in objs}
        for det in detections[scene_im_id]:
            score = det.get("score", 1.0)
            if score < score_thr:
                continue
            obj_name = id2obj.get(det["obj_id"], "unknown")
            if obj_name not in objs:
                continue
            if train_objs is not None and obj_name not in train_objs:
                continue
            obj_annotations[obj_name].append({"category_id": objs.index(obj_name), "bbox_est": det["bbox_est"], "score": score,
                                              "time": det.get("time", 0.0)})
        annotations = []
        for obj, cur in obj_annotations.items():
            scores = [a["score"] for a in cur]
            annotations.extend([a for _, a in sorted(zip(scores, cur), key=lambda p: p[0], reverse=True)][:top_k_per_obj])
        out.append((scene_im_id, annotations))
    return out


@pytest.mark.parametrize("thr,topk,train", [(0.0, 1, None), (0.3, 2, None), (0.5, 100, [5, 9]), (0.0, 3, [1])])
def test_detection_loading_matches_reference(thr, topk, train):
    obj_ids = G.DATASET_OBJ_IDS["lmo"]
    id2obj = {o: f"obj{o}" for o in obj_ids}
    images = [(2, i) for i in (1, 3, 5, 7, 9)]
    b = lambda k: [10.0 * k, 5.0, 20.5, 30.25]
    dets = {
        "2/1": [{"obj_id": 5, "bbox_est": b(1), "score": 0.9, "time": 0.1}, {"obj_id": 5, "bbox_est": b(2), "score": 0.9},
                {"obj_id": 5, "bbox_est": b(3), "score": 0.95}, {"obj_id": 1, "bbox_est": b(4), "score": 0.2},
                {"obj_id": 2, "bbox_est": b(5), "score": 0.99}, {"obj_id": 9, "bbox_est": b(6), "score": 0.5},
                {"obj_id": 9, "bbox_est": b(7), "score": 0.5}, {"obj_id": 12, "bbox_est": b(8), "score": 0.3}],
        "2/3": [],                                                     # kept, no ROIs
        "2/7": [{"obj_id": 1, "bbox_est": b(9), "score": 0.6}, {"obj_id": 99, "bbox_est": b(10), "score": 0.7},
                {"obj_id": 1, "bbox_est": b(11), "score": 0.6}, {"obj_id": 1, "bbox_est": b(12), "score": 0.6}],
        "2/9": [{"obj_id": 9, "bbox_est": b(13)}],                       # no score: 1.0
    }                                                                 # 2/5: missing -> skipped
    got = G.load_detections(dets, images, obj_ids, thr, topk, train)
    ref = _ref_load_detections(dets, [f"{s}/{i}" for s, i in images], [id2obj[o] for o in obj_ids], id2obj, thr, topk,
                               None if train is None else [id2obj[o] for o in train])
    assert [f"{images[i][0]}/{images[i][1]}" for i, _ in got] == [k for k, _ in ref]
    for (_, a), (_, r) in zip(got, ref):
        assert [(x["label"], x["bbox_est"], x["score"], x["time"]) for x in a] == \
               [(y["category_id"], y["bbox_est"], y["score"], y["time"]) for y in r]
        assert all(obj_ids[x["label"]] == x["obj_id"] for x in a)


def test_image_list_and_label_table():
    t = [{"scene_id": 3, "im_id": 2, "obj_id": 5}, {"scene_id": 1, "im_id": 9, "obj_id": 5}, {"scene_id": 3, "im_id": 2, "obj_id": 7},
         {"scene_id": 1, "im_id": 4, "obj_id": 1}]
    assert G.image_list(t) == [(1, 4), (1, 9), (3, 2)]
    shipped = {"lmo": 8, "hb": 16, "ycbv": 21, "tless": 30, "tudl": 3, "icbin": 2, "itodd": 28}
    assert {k: len(v) for k, v in G.DATASET_OBJ_IDS.items()} == shipped
    assert G.label_obj_ids("lmo") == [1, 5, 6, 8, 9, 10, 11, 12]
    assert G.label_obj_ids("other", t) == [1, 5, 7]


def test_pack_batches():
    rng = np.random.RandomState(0)
    for _ in range(200):
        counts = list(rng.randint(0, 12, rng.randint(1, 40)))
        mb = int(rng.choice([1, 5, 8, 64]))
        keys = list(rng.randint(0, 2, len(counts))) if rng.rand() < 0.3 else None
        batches = G.pack_batches(counts, mb, keys)
        assert [i for b in batches for i in b] == list(range(len(counts)))   # whole images, in order
        for b in batches:
            n = sum(counts[i] for i in b)
            assert n <= mb or len(b) == 1                                   # only an oversized image goes alone
            if keys is not None:
                assert len({keys[i] for i in b}) == 1
        for b0, b1 in zip(batches, batches[1:]):   # greedy: the next image did not fit (or changed size)
            nxt = b1[0]
            assert sum(counts[i] for i in b0) + counts[nxt] > mb or (keys is not None and keys[nxt] != keys[b0[0]])


def test_csv_name_and_exp_id():
    cfg = _cfg(USE_PNP=True, PNP_TYPE="ransac_pnp")
    e = G.exp_id(cfg, "configs/gdrn/ycbv/convnext_a6_AugCosyAAEGray_BG05_mlL1_DMask_amodalClipBox_classAware_ycbv.py")
    assert e == "convnext_a6_AugCosyAAEGray_BG05_mlL1_DMask_amodalClipBox_classAware_ycbvRANSAC_PNP_test"
    assert G.result_csv_name(cfg, e) == \
        "convnext-a6-AugCosyAAEGray-BG05-mlL1-DMask-amodalClipBox-classAware-ycbvRANSAC-PNP-test-iter0_ycbv-test.csv"
    cfg.TEST.USE_PNP = False
    cfg.VAL.SPLIT_TYPE = "bb8"
    assert G.exp_id(cfg, "a/b_c.py") == "b_c_test"
    assert G.result_csv_name(cfg, "b_c_test") == "b-c-test-iter0_ycbv-test-bb8.csv"


def test_time_column():
    images = [(1, 1), (1, 2), (2, 5)]
    imgs = [(0, [{"obj_id": 3, "score": 0.5, "time": 0.25}, {"obj_id": 4, "score": 0.7, "time": 9.0}]), (1, []),
            (2, [{"obj_id": 1, "score": 1.0, "time": 0.0}])]
    poses = np.arange(36, dtype=np.float32).reshape(3, 3, 4)
    rows = G.batch_rows(images, imgs, poses, 0.3)
    assert [(r["scene_id"], r["im_id"], r["obj_id"]) for r in rows] == [(1, 1, 3), (1, 1, 4), (2, 5, 1)]
    assert rows[0]["time"] == rows[1]["time"] == pytest.approx(0.35) and rows[2]["time"] == pytest.approx(0.1)
    assert np.array_equal(rows[1]["R"], poses[1, :, :3]) and np.array_equal(rows[2]["t"], poses[2, :, 3])


@pytest.mark.parametrize("setting,value,word", [
    ("TEST.TEST_BBOX_TYPE", "gt", "TEST.TEST_BBOX_TYPE"), ("TEST.COLOR_AUG", True, "TEST.COLOR_AUG"),
    ("MODEL.POSE_NET.PNP_NET.COORD_2D_TYPE", "rel", "COORD_2D_TYPE"),
    ("MODEL.POSE_NET.NAME", "GDRN_double_mask_depth", "MODEL.POSE_NET.NAME"), ("VAL.USE_BOP", False, "VAL.USE_BOP"),
    ("VAL.EVAL_CACHED", True, "VAL.EVAL_CACHED"), ("INPUT.MIN_SIZE_TEST", 400, "INPUT.MIN_SIZE_TEST")])
def test_rejections(setting, value, word):
    from gdrnpp_bop2022_b200.main_gdrn import set_opt

    cfg = _cfg()
    G.check_config(cfg, (480, 640))
    set_opt(cfg, setting, value)
    with pytest.raises(NotImplementedError, match=word.replace(".", r"\.")):
        G.check_config(cfg, (480, 640))


def test_shipped_resizes_are_identity():
    cfg = _cfg()
    G.check_config(cfg, (480, 640))
    cfg.INPUT.MIN_SIZE_TEST, cfg.INPUT.MAX_SIZE_TEST = 960, 1280
    G.check_config(cfg, (960, 1280))
    cfg.INPUT.MIN_SIZE_TEST, cfg.INPUT.MAX_SIZE_TEST, cfg.INPUT.IMG_AUG_RESIZE = 480, 640, False
    G.check_config(cfg, (540, 720))


def test_coord_grid_formula():
    """The kernel computes get_2d_coord_np's grid value as f32(k * (1.0 / n)) in float64: np.linspace's arithmetic."""
    for n in (1, 3, 7, 480, 540, 640, 720, 960, 1080, 1280, 1920):
        k = np.arange(n)
        assert np.array_equal(np.linspace(0, 1, n, endpoint=False, dtype=np.float32), (k * (1.0 / n)).astype(np.float32))


def test_cli_opts():
    from gdrnpp_bop2022_b200.main_gdrn import parse_opts

    o, w = parse_opts(["MODEL.WEIGHTS=out/model_final.pth", "INPUT.WITH_DEPTH=True", "TEST.USE_DEPTH_REFINE=True"])
    assert o == {"MODEL.WEIGHTS": "out/model_final.pth", "INPUT.WITH_DEPTH": True, "TEST.USE_DEPTH_REFINE": True} and w is None
    o, w = parse_opts(["MODEL.WEIGHTS=1=a.pth", "5=b.pth", "TEST.USE_PNP=False"])
    assert w == {1: "a.pth", 5: "b.pth"} and o == {"TEST.USE_PNP": False}


# ---------------------------------------------------------------------------------------------------- GPU
def _host_roi_setup(xywh, H, W, dzi, in_res=256, out_res=64):
    """read_data_test (data_loader.py:751-769) + batch_data_test (engine_utils.py:213-241) for one detection."""
    from gdrnpp_bop2022_b200.native_ops import get_affine_transform

    arr = torch.tensor([list(xywh)])
    arr[:, 2] += arr[:, 0]
    arr[:, 3] += arr[:, 1]
    x1, y1, x2, y2 = np.array(arr.flatten().tolist())            # BoxMode.convert -> list -> apply_box (float64)
    bbox_center = np.array([0.5 * (x1 + x2), 0.5 * (y1 + y2)])
    bw, bh = max(x2 - x1, 1), max(y2 - y1, 1)
    scale = min(max(bh, bw) * dzi, max(H, W)) * 1.0
    M_in = get_affine_transform(bbox_center, (scale, scale), 0, (in_res, in_res))   # crop_resize_by_warp_affine's tuple
    M_out = get_affine_transform(bbox_center, (scale, scale), 0, (out_res, out_res))
    return {"roi_center": bbox_center.astype(np.float32), "roi_wh": np.array([bw, bh], np.float32),
            "scale": np.float32(scale), "resize_ratio": np.float32(out_res / scale), "bbox_est": np.float32([x1, y1, x2, y2]),
            "M_in": M_in.reshape(6), "M_out": M_out.reshape(6)}


def _random_dets(rng, N, H, W, n, nc):
    meta, xywh = [], []
    for i in range(n):
        kind = i % 4
        w, h = rng.uniform(5, 300, 2)
        if kind == 1:
            w, h = rng.uniform(0.1, 0.99), rng.uniform(0.1, 3)        # w or h < 1
        if kind == 2:
            w, h = rng.uniform(500, 1500, 2)                          # scale clamped by max(H, W)
        x, y = rng.uniform(-w / 2, W - w / 2), rng.uniform(-h / 2, H - h / 2)   # often partly outside
        meta.append((rng.randint(N), rng.randint(nc)))
        xywh.append((float(x), float(y), float(w), float(h)))
    return meta, xywh


def _run_inputs(dev, images, meta, xywh, Ks, extents, depth=None, factor=None, dzi=1.5):
    from gdrnpp_bop2022_b200.native_ops import roi_batch_inputs

    dets = {"det_meta": torch.tensor(meta, dtype=torch.int32, device=dev),
            "bbox_est": torch.tensor(np.asarray(xywh, np.float32), device=dev)}
    return roi_batch_inputs(images, dets, Ks, extents, dzi, depth=depth, depth_factor=factor)


@pytest.mark.gpu
def test_roi_setup_matches_loader(dev):
    rng = np.random.RandomState(1)
    H, W, N, nc = 480, 640, 3, 5
    meta, xywh = _random_dets(rng, N, H, W, 200, nc)
    Ks = torch.tensor(rng.uniform(100, 600, (N, 3, 3)), dtype=torch.float32, device=dev)
    ext = torch.tensor(rng.uniform(0.01, 0.3, (nc, 3)), dtype=torch.float32, device=dev)
    images = torch.zeros((N, H, W, 3), dtype=torch.uint8, device=dev)
    out = {k: v.cpu().numpy() for k, v in _run_inputs(dev, images, meta, xywh, Ks, ext).items()}
    for i, ((img, lab), b) in enumerate(zip(meta, xywh)):
        ref = _host_roi_setup(b, H, W, 1.5)
        for k in ("roi_center", "roi_wh", "scale", "resize_ratio", "bbox_est"):
            assert np.array_equal(out[k][i], ref[k]), (i, k, out[k][i], ref[k])
        for k in ("M_in", "M_out"):
            np.testing.assert_allclose(out[k][i], ref[k], rtol=1e-12, atol=1e-12 * np.abs(ref[k]).max())
        assert out["roi_cls"][i] == lab and out["roi_cls"].dtype == np.int64
        assert np.array_equal(out["roi_extent"][i], ext[lab].cpu().numpy())
        assert np.array_equal(out["roi_cam"][i], Ks[img].cpu().numpy())
        assert out["im_H"][i] == H and out["im_W"][i] == W
    assert (out["scale"] == max(H, W)).sum() > 10 and (out["roi_wh"] == 1).sum() > 10


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,C", [(1, 480, 640, 3), (4, 480, 640, 3), (9, 480, 640, 3), (2, 960, 1280, 1)])
def test_roi_crop_multi_matches_per_image(dev, N, H, W, C):
    from gdrnpp_bop2022_b200.native_ops import crop_resize_float, crop_resize_image

    rng = np.random.RandomState(N * 7 + C)
    meta, xywh = _random_dets(rng, N, H, W, 5 * N + 3, 4)
    imgs = rng.randint(0, 256, (N, H, W, C)).astype(np.uint8)
    depth = rng.randint(0, 65536, (N, H, W)).astype(np.uint16)
    factor = rng.choice([1.0, 10.0, 1000.0 / 0.1], N)
    Ks = torch.eye(3, device=dev).expand(N, 3, 3).contiguous()
    ext = torch.ones((4, 3), device=dev)
    out = _run_inputs(dev, torch.from_numpy(imgs).to(dev), meta, xywh, Ks, ext, torch.from_numpy(depth).to(dev),
                      torch.from_numpy(factor).to(dev))
    xs = np.linspace(0, 1, W, endpoint=False, dtype=np.float32)
    ys = np.linspace(0, 1, H, endpoint=False, dtype=np.float32)
    grid = torch.from_numpy(np.ascontiguousarray(np.asarray(np.meshgrid(xs, ys)).transpose(1, 2, 0))).to(dev)
    for i, (img, _) in enumerate(meta):
        Mi, Mo = out["M_in"][i:i + 1], out["M_out"][i:i + 1]
        im3 = np.repeat(imgs[img], 3, axis=2) if C == 1 else imgs[img]   # cv2.imread(IMREAD_COLOR) of a gray image
        ref_img = crop_resize_image(torch.from_numpy(np.ascontiguousarray(im3)).to(dev), Mi, 256)
        assert torch.equal(out["roi_img"][i:i + 1], ref_img), i
        assert torch.equal(out["roi_coord_2d"][i:i + 1], crop_resize_float(grid, Mo, 64)), i
        d_m = torch.from_numpy((depth[img] / factor[img]).astype(np.float32)).to(dev)   # mmcv.imread / factor, astype f32
        ref_d = crop_resize_float(d_m, Mi, 256, nearest=True)
        assert torch.equal(out["roi_depth"][i:i + 1], ref_d), i
        d = ref_d[:, 0]
        sensor = ((d[:, 1::4, 1::4] + d[:, 1::4, 2::4]) + (d[:, 2::4, 1::4] + d[:, 2::4, 2::4])) * 0.25   # GdrnPredictor
        assert torch.equal(out["depth_sensor"][i:i + 1], sensor), i


def _tree(tmp_path, **kw):
    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    root = str(tmp_path / "datasets")
    det = write_bop_tree(root, **kw)
    return root, det


def _model(cfg, dev, precision="bf16x3", num_classes=21, seed=0, max_batch=64):
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    m = GDRN_DoubleMask(cfg, max_batch=max_batch, precision=precision)
    m.load_state_dict(make_state_dict(num_classes=num_classes, seed=seed))
    return m.to(dev)


def _angle(Ra, Rb):
    """Rotation difference in rad, as the parity tests measure it (well conditioned at 0, unlike arccos of the trace)."""
    return 2 * np.arcsin(np.minimum(np.linalg.norm((Ra - Rb).reshape(len(Ra), -1), axis=1) / (2 * 2 ** 0.5), 1.0))


def _compare(a, b, ang_tol, t_tol):
    assert [(r["scene_id"], r["im_id"], r["obj_id"], r["score"]) for r in a] == \
           [(r["scene_id"], r["im_id"], r["obj_id"], r["score"]) for r in b]
    Ra, Rb = np.stack([r["R"] for r in a]), np.stack([r["R"] for r in b])
    ta, tb = np.stack([r["t"] for r in a]), np.stack([r["t"] for r in b])
    ang, terr = _angle(Ra, Rb).max(), np.abs(ta - tb).max()
    assert ang < ang_tol and terr < t_tol, (ang, terr)
    return bool(np.array_equal(Ra, Rb) and np.array_equal(ta, tb)), ang, terr


@pytest.mark.gpu
@pytest.mark.parametrize("precision,ang_tol,t_tol", [("bf16x3", 1e-4, 1e-3), ("bf16", 0.1, 1e-2)])
def test_batched_equals_one_image_per_forward(dev, tmp_path, precision, ang_tol, t_tol):
    root, det = _tree(tmp_path, num_images=14, seed=3)
    cfg = _cfg(det)
    model = _model(cfg, dev, precision)
    a = G.gdrn_inference_on_dataset(cfg, model, root, max_batch=64)
    b = G.gdrn_inference_on_dataset(cfg, model, root, max_batch=1)
    assert len(a) > 40
    bitwise, ang, terr = _compare(a, b, ang_tol, t_tol)
    print(f"{precision}: max_batch 64 vs 1 bitwise equal: {bitwise} (max angle {ang:.2e} rad, max |dt| {terr:.2e} m)")


@pytest.mark.gpu
@pytest.mark.parametrize("pnp_type", ["ransac_pnp", "net_iter_pnp", "net_ransac_pnp", "net_ransac_pnp_rot"])
def test_use_pnp_ignores_depth_refine(dev, tmp_path, pnp_type):
    root, det = _tree(tmp_path, num_images=6, seed=4)
    cfg = _cfg(det, USE_PNP=True, PNP_TYPE=pnp_type, USE_DEPTH_REFINE=False)
    model = _model(cfg, dev)
    a = G.gdrn_inference_on_dataset(cfg, model, root)
    cfg.TEST.USE_DEPTH_REFINE = True
    cfg.INPUT.WITH_DEPTH = True
    b = G.gdrn_inference_on_dataset(cfg, model, root)
    assert _compare(a, b, 1e-6, 1e-6)[0]   # the same poses, bit for bit


def _per_image_driver(cfg, model, root, ts, dev):
    """The existing single-image calls: host get_affine_transform per ROI, three crop_resize launches per image, the
    host depth conversion, the forward, and depth refine on GdrnPredictor's sensor crop."""
    from gdrnpp_bop2022_b200.native_ops import crop_resize_float, crop_resize_image, get_affine_transform
    from gdrnpp_bop2022_b200.renderer import depth_refine, get_K_crop_resize

    meshes = ts.meshes(dev)
    info = json.load(open(os.path.join(ts.base, "models_eval", "models_info.json")))
    rows = []
    for idx, anns in ts.records:
        if not anns:
            continue
        im = G.read_image(ts.rgb[idx])
        H, W = im.shape[:2]
        d = (G.read_depth(ts.depth[idx]) / ts.depth_factor[idx]).astype(np.float32)
        s = [_host_roi_setup(a["bbox_est"], H, W, 1.5) for a in anns]
        n = len(anns)
        Min = np.stack([x["M_in"] for x in s])
        Mout = np.stack([x["M_out"] for x in s])
        roi_img = crop_resize_image(torch.from_numpy(im).to(dev), Min, 256)
        xs = np.linspace(0, 1, W, endpoint=False, dtype=np.float32)
        ys = np.linspace(0, 1, H, endpoint=False, dtype=np.float32)
        grid = torch.from_numpy(np.ascontiguousarray(np.asarray(np.meshgrid(xs, ys)).transpose(1, 2, 0))).to(dev)
        c2d = crop_resize_float(grid, Mout, 64)
        rd = crop_resize_float(torch.from_numpy(d).to(dev), Min, 256, nearest=True)[:, 0]
        f = lambda k: torch.from_numpy(np.stack([x[k] for x in s])).to(dev)
        cls = torch.tensor([a["label"] for a in anns], device=dev)
        cam = torch.from_numpy(ts.K[idx]).to(dev).expand(n, 3, 3).contiguous()
        ext = torch.tensor([[info[str(a["obj_id"])]["size_" + c] / 1000.0 for c in "xyz"] for a in anns],
                           dtype=torch.float32, device=dev)
        out = model(roi_img, roi_classes=cls, roi_coord_2d=c2d, roi_cams=cam, roi_centers=f("roi_center"),
                    roi_whs=f("roi_wh"), roi_extents=ext, resize_ratios=f("resize_ratio"))
        scale = f("scale")
        K_crop = get_K_crop_resize(cam, f("roi_center") - scale.view(n, 1) / 2, (64.0 / scale).view(n, 1))
        sensor = ((rd[:, 1::4, 1::4] + rd[:, 1::4, 2::4]) + (rd[:, 2::4, 1::4] + rd[:, 2::4, 2::4])) * 0.25
        xyz = torch.cat([out["coor_x"], out["coor_y"], out["coor_z"]], dim=1)
        t = depth_refine(meshes, out["rot"], out["trans"], K_crop, xyz, out["mask"], sensor.contiguous(),
                         iters=cfg.TEST.DEPTH_REFINE_ITER, thresh=cfg.TEST.DEPTH_REFINE_THRESHOLD, mesh_ids=cls,
                         coor_z_refine=cfg.TEST.USE_COOR_Z_REFINE)
        R = out["rot"].cpu().numpy()
        t = t.cpu().numpy()
        sid, iid = ts.images[idx]
        for k, a in enumerate(anns):
            rows.append({"scene_id": sid, "im_id": iid, "obj_id": a["obj_id"], "score": float(np.float32(a["score"])),
                         "R": R[k].astype(np.float64), "t": t[k].astype(np.float64)})
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("coor_z", [False, True])
def test_depth_refine_matches_per_image_model3d_driver(dev, tmp_path, coor_z):
    root, det = _tree(tmp_path, num_images=6, seed=5)
    cfg = _cfg(det, USE_PNP=False, USE_DEPTH_REFINE=True, USE_COOR_Z_REFINE=coor_z, DEPTH_REFINE_ITER=2,
               DEPTH_REFINE_THRESHOLD=0.8)
    cfg.INPUT.WITH_DEPTH = True
    model = _model(cfg, dev)
    ts = G.TestSet(cfg, root)
    a = G.gdrn_inference_on_dataset(cfg, model, root, test_set=ts)
    b = _per_image_driver(cfg, model, root, ts, dev)
    bitwise, ang, terr = _compare(a, b, 1e-4, 1e-3)
    print(f"depth refine (coor_z={coor_z}) vs per-image driver: bitwise {bitwise}, angle {ang:.2e}, |dt| {terr:.2e}")


@pytest.mark.gpu
def test_per_object_one_pass(dev, tmp_path):
    root, det = _tree(tmp_path, num_images=8, seed=6, dets_per_image=21)   # every object in every image
    cfg = _cfg(det)
    g = cfg.MODEL.POSE_NET.GEO_HEAD
    g.XYZ_CLASS_AWARE = g.MASK_CLASS_AWARE = g.REGION_CLASS_AWARE = False
    cfg.MODEL.POSE_NET.NUM_CLASSES = 1
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    objs = [2, 5, 11]
    sds = {o: make_state_dict(num_classes=1, seed=40 + o) for o in objs}
    ts = G.TestSet(cfg, root, objs)
    both = G.gdrn_inference_on_dataset(cfg, G.build_model(cfg, sds, obj_ids=ts.obj_ids), root, train_obj_ids=objs)
    per = []
    for o in objs:
        m = G.build_model(cfg, sds[o])
        per += G.gdrn_inference_on_dataset(cfg, m, root, train_obj_ids=[o])
    key = {(s, i): k for k, (s, i) in enumerate(ts.images)}
    per = sorted(per, key=lambda r: key[(r["scene_id"], r["im_id"])])   # stable: object (label) order within an image
    assert len(both) == len(per) > 10
    _compare(both, per, 1e-4, 1e-3)


@pytest.mark.gpu
def test_scoring_matches_script(dev, tmp_path):
    from gdrnpp_bop2022_b200 import bop_eval
    from gdrnpp_bop2022_b200 import eval_pose_results_more as E

    root, det = _tree(tmp_path, num_images=6, seed=7)
    cfg = _cfg(det)
    model = _model(cfg, dev)
    rows = G.gdrn_inference_on_dataset(cfg, model, root)
    out1 = str(tmp_path / "eval_a")
    res = G.GdrnDatasetEvaluator(cfg, root, out1, "cfg_test").evaluate(rows)
    loaded = bop_eval.load_bop_results(res["csv"])
    assert len(loaded) == len(rows)
    assert all(abs(a["t"].reshape(3) - 1000 * b["t"]).max() < 1e-3 for a, b in zip(loaded, rows))
    out2 = str(tmp_path / "eval_b")
    os.makedirs(out2)
    name = os.path.basename(res["csv"])
    import shutil

    shutil.copy(res["csv"], os.path.join(out2, name))
    E.run(E.parse_args(["--results_path", out2, "--result_filenames", name, "--error_types", "ad,reteS,proj",
                        "--eval_path", out2, "--n_top", "-1", "--datasets_path", os.path.join(root, "BOP_DATASETS")]))
    for dp, _, files in os.walk(out1):
        for f in files:
            if f.endswith(".json"):
                rel = os.path.relpath(os.path.join(dp, f), out1)
                assert open(os.path.join(dp, f)).read() == open(os.path.join(out2, rel)).read(), rel
