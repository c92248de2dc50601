"""The save-results loop (gdrn_evaluator.gdrn_save_result_of_dataset, main_gdrn TEST.SAVE_RESULTS_ONLY), its mask
kernels (csrc/mask_rle.cu: paste, RLE encode, RLE decode + confusion counts) and the mask tools (mask_metrics.py)."""
import os
import pickle
import pickletools
import types

import numpy as np
import pytest
import torch

from gdrnpp_bop2022_b200 import gdrn_evaluator as G
from gdrnpp_bop2022_b200.gdrn_model import default_cfg
from oracle import mask_oracle as MO


def _cfg(det_file="datasets/none.json", dataset="ycbv", **test):
    cfg = default_cfg(with_maps=False)
    cfg.VAL = types.SimpleNamespace(DATASET_NAME=dataset, SPLIT="test", SPLIT_TYPE="", TARGETS_FILENAME="test_targets_bop19.json",
                                    USE_BOP=True, EVAL_CACHED=False)
    cfg.DATASETS = types.SimpleNamespace(TEST=(f"{dataset}_bop_test",), DET_FILES_TEST=(det_file,), DET_THR=0.0,
                                         DET_TOPK_PER_OBJ=100)
    cfg.INPUT = types.SimpleNamespace(WITH_DEPTH=False, DZI_PAD_SCALE=1.5, MIN_SIZE_TEST=480, MAX_SIZE_TEST=640)
    cfg.TEST.SAVE_RESULTS_ONLY = True
    for k, v in test.items():
        setattr(cfg.TEST, k, v)
    return cfg


# ---------------------------------------------------------------------------------------------------- CPU: oracle
def _edge_masks(rng):
    out = [np.zeros((5, 7), bool), np.ones((5, 7), bool), np.zeros((1, 1), bool), np.ones((1, 1), bool)]
    m = np.zeros((6, 4), bool)
    m[0, 0] = True                                   # pixel (0,0): the first count is 0
    out.append(m)
    out.append(rng.rand(1, 50) < 0.5)                # single-pixel columns
    out.append(rng.rand(50, 1) < 0.5)
    big = np.zeros((1000, 1100), bool)               # counts of ~10^6: five chars
    big[500:, 700:] = True
    out.append(big)
    for _ in range(30):
        h, w = rng.randint(1, 40, 2)
        out.append(rng.rand(h, w) < rng.uniform(0.05, 0.95))
    return out


def test_oracle_rle_roundtrip():
    rng = np.random.RandomState(0)
    for m in _edge_masks(rng):
        counts = MO.rle_encode(m)
        assert sum(counts) == m.size
        s = MO.rle_to_string(counts)
        assert MO.rle_fr_string(s) == counts
        assert np.array_equal(MO.rle_decode(counts, *m.shape), m.astype(np.uint8))
        assert np.array_equal(MO.decode(MO.encode(m)), m.astype(np.uint8))
    assert MO.rle_encode(np.zeros((5, 7))) == [35] and MO.rle_encode(np.ones((5, 7))) == [0, 35]
    big = _edge_masks(rng)[7]
    assert max(len(MO.rle_to_string([c])) for c in MO.rle_encode(big)) >= 5


def test_oracle_rle_hand_worked():
    assert MO.rle_to_string([4]) == "4"                       # 2x2 empty
    assert MO.rle_to_string([0, 4]) == "04"                   # 2x2 full
    assert MO.encode(np.array([[1, 0], [0, 0]])) == {"size": [2, 2], "counts": "013"}
    assert MO.rle_to_string([16]) == "`0"                     # 16 = 0b10000: a second group keeps the sign positive
    col = np.array([[0], [1], [1], [1], [1], [1], [0], [1]])
    assert MO.rle_encode(col) == [1, 5, 1, 1]
    assert MO.encode(col)["counts"] == "151L"                 # 1 - cnts[1] = -4 -> 0x1c + 48
    assert MO.rle_fr_string("151L") == [1, 5, 1, 1]


def _np_paste(prob, box, H, W):
    """Bilinear paste in float64 from the definition (pixel centres, align_corners=False, zero padding)."""
    M = prob.shape[0]
    x0, y0, x1, y1 = [float(v) for v in box]
    xs = ((np.arange(W) + 0.5 - x0) / (x1 - x0)) * M - 0.5
    ys = ((np.arange(H) + 0.5 - y0) / (y1 - y0)) * M - 0.5
    pad = np.zeros((M + 2, M + 2))
    pad[1:-1, 1:-1] = prob
    fx, fy = np.floor(xs), np.floor(ys)
    ax, ay = xs - fx, ys - fy
    ix = np.clip(fx.astype(np.int64) + 1, 0, M + 1)
    iy = np.clip(fy.astype(np.int64) + 1, 0, M + 1)
    ix1, iy1 = np.clip(ix + 1, 0, M + 1), np.clip(iy + 1, 0, M + 1)
    okx, oky = (fx >= -1) & (fx <= M - 1), (fy >= -1) & (fy <= M - 1)
    v = ((1 - ay)[:, None] * (1 - ax)[None] * pad[iy][:, ix] + (1 - ay)[:, None] * ax[None] * pad[iy][:, ix1]
         + ay[:, None] * (1 - ax)[None] * pad[iy1][:, ix] + ay[:, None] * ax[None] * pad[iy1][:, ix1])
    return v * (oky[:, None] & okx[None])


def test_oracle_paste_matches_definition():
    rng = np.random.RandomState(1)
    H, W = 48, 64
    probs = torch.from_numpy(rng.rand(6, 16, 16).astype(np.float32))
    boxes = torch.tensor([[5, 6, 30, 40], [-10, -3, 20, 15], [50, 30, 80, 70], [10.3, 10.1, 10.8, 10.5],
                          [-20, -30, 100, 90], [2.5, 3.25, 47.75, 44.5]], dtype=torch.float32)
    got = MO.paste_masks(probs, boxes, (H, W), 0.5).numpy()
    for i in range(6):
        ref = _np_paste(probs[i].double().numpy(), boxes[i].numpy(), H, W)
        far = np.abs(ref - 0.5) > 1e-4
        assert np.array_equal(got[i][far], (ref >= 0.5)[far]), i
        assert far.mean() > 0.99


def test_metric_restatements_hand_cases():
    from gdrnpp_bop2022_b200.mask_metrics import metrics_from_counts

    z, o = np.zeros((4, 5), bool), np.ones((4, 5), bool)
    some = z.copy()
    some[1:3, 2:4] = True
    cases = [(z, z, 1.0, 0.0),          # all-zero GT, empty prediction: only the background label, F1 0 / 0 -> 0
             (o, o, 1.0, 1.0),          # all-one GT, full prediction
             (z, o, 0.0, 0.0),          # all-one GT, empty prediction
             (z, some, 0.5 * (16 / 20), 0.0),   # empty prediction: background IoU 16/20, object IoU 0
             (o, z, 0.0, 0.0)]
    for pred, gt, miou, f1 in cases:
        assert MO.compute_mean_iou(pred, gt) == pytest.approx(miou)
        assert MO.f1_binary(pred, gt) == pytest.approx(f1)
        p, g = pred.ravel(), gt.ravel()
        c = [[np.sum(p & g), np.sum(p & ~g), np.sum(~p & g), np.sum(~p & ~g)]]
        m, f = metrics_from_counts(c)
        assert m[0] == pytest.approx(miou) and f[0] == pytest.approx(f1)
    rng = np.random.RandomState(2)
    for _ in range(50):
        pred, gt = rng.rand(6, 7) < rng.rand(), rng.rand(6, 7) < rng.rand()
        p, g = pred.ravel(), gt.ravel()
        m, f = metrics_from_counts([[np.sum(p & g), np.sum(p & ~g), np.sum(~p & g), np.sum(~p & ~g)]])
        assert m[0] == pytest.approx(MO.compute_mean_iou(pred, gt)) and f[0] == pytest.approx(MO.f1_binary(pred, gt))


# ---------------------------------------------------------------------------------------------------- CPU: results.pkl
def test_save_record_dtypes_and_box():
    det = {"obj_id": 5, "score": 0.7, "bbox_est": [10.1, 20.3, 33.7, 0.45]}
    pose = np.arange(12, dtype=np.float32).reshape(3, 4)
    m, fm = {"size": [2, 2], "counts": "4"}, {"size": [2, 2], "counts": "04"}
    r = G.save_record(det, pose, m, fm, use_pnp=False)
    assert r["R"].dtype == np.float32 and r["t"].dtype == np.float32
    assert np.array_equal(r["R"], pose[:, :3]) and np.array_equal(r["t"], pose[:, 3])
    arr = torch.tensor([det["bbox_est"]])                      # BoxMode.convert XYWH -> XYXY through float32
    arr[:, 2] += arr[:, 0]
    arr[:, 3] += arr[:, 1]
    assert r["bbox_est"].dtype == np.float32 and np.array_equal(r["bbox_est"], arr[0].numpy())
    assert r["score"] == float(np.float32(0.7)) and type(r["score"]) is float
    assert r["mask"] is m and r["full_mask"] is fm and r["obj_id"] == 5
    p = G.save_record(det, pose, m, fm, use_pnp=True)
    assert p["R"].dtype == np.float64 and p["t"].dtype == np.float64 and np.array_equal(p["R"], pose[:, :3])
    s = G.save_record(det, np.full((3, 4), -100, np.float32), m, fm, use_pnp=True)
    assert s["R"].dtype == np.float32 and (s["t"] == -100).all()


def test_results_dict_and_pickle(tmp_path):
    rows = [("1/4", {"obj_id": 3}), ("1/4", {"obj_id": 1}), ("2/1", {"obj_id": 7}), ("1/10", {"obj_id": 2})]
    d = G.results_dict(rows)
    assert list(d) == ["1/4", "2/1", "1/10"] and [r["obj_id"] for r in d["1/4"]] == [3, 1]
    path = G.write_results_pkl(d, str(tmp_path / "out"))
    assert path == str(tmp_path / "out" / "results.pkl")
    raw = open(path, "rb").read()
    assert next(pickletools.genops(raw))[0].name == "PROTO" and raw[:2] == b"\x80\x02"
    assert pickle.loads(raw) == d


def test_output_dir_naming_and_single_test_dataset():
    cfg = _cfg(dataset="lmo")
    cfg.OUTPUT_DIR = "output/gdrn/lmo_pbr/cfg"
    cfg.MODEL.WEIGHTS = "output/gdrn/lmo_pbr/cfg/model_final_wo_optim-e8c99c96.pth"
    assert G.save_results_dir(cfg) == "output/gdrn/lmo_pbr/cfg/inference_model_final_wo_optim-e8c99c96/lmo_bop_test"
    cfg.MODEL.WEIGHTS = "a/b/model.final.pth"
    assert G.save_results_dir(cfg) == "output/gdrn/lmo_pbr/cfg/inference_model/lmo_bop_test"
    assert G.save_results_dir(cfg, per_object=True) == "output/gdrn/lmo_pbr/cfg/inference_per_object/lmo_bop_test"
    cfg.DATASETS.TEST = ("lmo_bop_test", "ycbv_bop_test")
    with pytest.raises(ValueError, match="exactly one DATASETS.TEST"):
        G.save_results_dir(cfg)


def test_threshold_must_be_positive(lib):
    from gdrnpp_bop2022_b200 import native_ops

    for thr in (0.0, -0.5, float("nan")):
        with pytest.raises(ValueError, match="threshold must be > 0"):
            native_ops.paste_masks_in_image(torch.zeros(1, 4, 4), torch.zeros(1, 4), (8, 8), thr)
        with pytest.raises(ValueError, match="threshold must be > 0"):
            native_ops.paste_masks_rle_launch(torch.zeros(1, 1, 4, 4), None, torch.zeros(1, 2), torch.ones(1), (8, 8), thr, "L1")
        # the C entries reject it before touching any pointer
        assert lib.gdrn_mask_paste(None, 1, 4, 4, 0, None, 8, 8, thr, None, None) != 0
        assert b"threshold must be > 0" in lib.gdrn_last_error()
        assert lib.gdrn_mask_paste_rle(None, None, 1, 4, 4, 1, None, None, 8, 8, thr, None, 0, None, 0, None, None) != 0


# ---------------------------------------------------------------------------------------------------- GPU: kernels
def _maps(rng, n, kind, M=64):
    x = rng.randn(n, 1, M, M).astype(np.float32) * 2
    if kind == "L1":
        x[0] = 0.25                                              # a constant map: NaN probabilities, pastes to 0
    return torch.from_numpy(x)


def _boxes(rng, n, H, W):
    """roi_center / scale covering: inside, partly and wholly outside, smaller than a pixel, larger than the image."""
    c = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
    s = rng.uniform(20, 300, n)
    for i in range(n):
        k = i % 6
        if k == 1:
            c[i] = [rng.uniform(-60, 0), rng.uniform(H, H + 60)]      # partly outside
        elif k == 2:
            c[i] = [W + 500, rng.uniform(0, H)]                       # wholly outside
        elif k == 3:
            s[i] = rng.uniform(0.1, 0.9)                              # smaller than a pixel
        elif k == 4:
            s[i] = rng.uniform(1.2, 2.5) * max(H, W)                  # larger than the image
    return torch.tensor(c, dtype=torch.float32), torch.tensor(s, dtype=torch.float32)


PASTE_CASES = [(n, H, W, kind, thr) for n in (1, 5, 64) for (H, W) in ((480, 640), (960, 1280))
               for kind in ("L1", "BCE") for thr in (0.5, 0.3) if not (n == 64 and H == 960 and thr == 0.3)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,H,W,kind,thr", PASTE_CASES)
def test_paste_and_rle_match_detectron2_path(dev, n, H, W, kind, thr):
    from gdrnpp_bop2022_b200 import native_ops

    rng = np.random.RandomState(n * 31 + H + int(thr * 10) + len(kind))
    raw = _maps(rng, n, kind).to(dev)
    center, scale = (t.to(dev) for t in _boxes(rng, n, H, W))
    prob = MO.get_out_mask(raw, kind)
    boxes = MO.inst_rois(center, scale)
    ref = MO.paste_masks(prob[:, 0], boxes, (H, W), thr)
    got = native_ops.paste_masks_in_image(prob[:, 0], boxes, (H, W), thr)
    assert got.dtype == torch.bool and torch.equal(got, ref)
    rles = native_ops.paste_masks_rle(raw, center, scale, (H, W), thr, kind)
    ref_np = ref.cpu().numpy()
    assert [r["counts"] for r in rles] == [MO.encode(m)["counts"] for m in ref_np]
    assert all(r["size"] == [H, W] for r in rles)
    assert ref_np.any(axis=(1, 2)).sum() >= min(n, 2) - 1


@pytest.mark.gpu
def test_rle_many_runs_per_column(dev):
    from gdrnpp_bop2022_b200 import native_ops

    H, W = 480, 640
    yy, xx = np.mgrid[0:64, 0:64]
    maps = [((yy + xx) % 2).astype(np.float32), ((yy // 2 + xx // 3) % 2).astype(np.float32), (yy % 2).astype(np.float32)]
    raw = torch.from_numpy(np.stack(maps)[:, None] * 4 - 2).to(dev)
    center = torch.tensor([[320.0, 240.0], [100.0, 0.0], [639.0, 479.0]], device=dev)
    scale = torch.tensor([600.0, 900.0, 200.0], device=dev)   # 9+ pixels per texel: many short runs per column
    for kind, thr in (("L1", 0.5), ("BCE", 0.3)):
        ref = MO.paste_masks(MO.get_out_mask(raw, kind)[:, 0], MO.inst_rois(center, scale), (H, W), thr).cpu().numpy()
        rles = native_ops.paste_masks_rle(raw, center, scale, (H, W), thr, kind)
        assert [r["counts"] for r in rles] == [MO.encode(m)["counts"] for m in ref]
        assert min(len(MO.rle_encode(m)) for m in ref) > 2000


@pytest.mark.gpu
def test_rle_confusion_counts_and_rejections(dev):
    from gdrnpp_bop2022_b200 import _lib, native_ops

    rng = np.random.RandomState(3)
    H, W = 37, 53
    preds = [rng.rand(H, W) < rng.uniform(0.05, 0.95) for _ in range(20)]
    preds += [np.zeros((H, W), bool), np.ones((H, W), bool)]
    gts = [rng.rand(H, W) < rng.uniform(0.05, 0.95) for _ in range(20)] + [np.ones((H, W), bool), np.zeros((H, W), bool)]
    rles = [MO.encode(p) for p in preds]
    got = native_ops.rle_confusion(rles, np.stack(gts).astype(np.uint8) * 7, device=dev)
    ref = [[np.sum(p & g), np.sum(p & ~g), np.sum(~p & g), np.sum(~p & ~g)] for p, g in zip(preds, gts)]
    assert got.dtype == np.int64 and np.array_equal(got, np.array(ref))
    good = MO.encode(preds[0])
    bad = {"total short of H*W": good["counts"][:-1],
           "unterminated group": good["counts"] + "`",
           "char outside the alphabet": good["counts"][:3] + "~" + good["counts"][3:],
           "total past H*W": good["counts"] + "9", "empty": ""}
    for why, s in bad.items():
        with pytest.raises(_lib.GdrnError, match="rle_confusion: string 1 is malformed"):
            native_ops.rle_confusion([good, {"size": [H, W], "counts": s}], np.stack(gts[:2]), device=dev)
    # the error channel does not poison the next call
    assert np.array_equal(native_ops.rle_confusion([good], gts[0][None], device=dev), np.array(ref[:1]))


# ---------------------------------------------------------------------------------------------------- GPU: the loop
def _tree(tmp_path, **kw):
    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    root = str(tmp_path / "datasets")
    return root, write_bop_tree(root, with_masks=True, **kw)


def _model(cfg, dev, precision="bf16x3", num_classes=21, seed=0, max_batch=64):
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    m = GDRN_DoubleMask(cfg, max_batch=max_batch, precision=precision)
    m.load_state_dict(make_state_dict(num_classes=num_classes, seed=seed))
    return m.to(dev)


def _per_image_driver(cfg, model, ts, dev):
    """One image per call: the ROI-input kernels, the forward, the torch paste of both masks, the oracle's RLE and the
    pose of step 6 (pnp_ransac_from_maps or the network's)."""
    from gdrnpp_bop2022_b200.native_ops import roi_batch_inputs
    from gdrnpp_bop2022_b200.pnp_ransac import pnp_ransac_from_maps

    out = {}
    thr = cfg.MODEL.POSE_NET.GEO_HEAD.MASK_THR_TEST
    for idx, anns in ts.records:
        if not anns:
            continue
        im = G.read_image(ts.rgb[idx])
        H, W = im.shape[:2]
        dets = {"det_meta": torch.tensor([[0, a["label"]] for a in anns], dtype=torch.int32, device=dev),
                "bbox_est": torch.tensor(np.asarray([a["bbox_est"] for a in anns], np.float32), device=dev)}
        inp = roi_batch_inputs(torch.from_numpy(im[None]).to(dev), dets, torch.from_numpy(ts.K[idx][None]).to(dev),
                               ts.extents(dev))
        o = model(inp["roi_img"], roi_classes=inp["roi_cls"], roi_coord_2d=inp["roi_coord_2d"], roi_cams=inp["roi_cam"],
                  roi_centers=inp["roi_center"], roi_whs=inp["roi_wh"], roi_extents=inp["roi_extent"],
                  resize_ratios=inp["resize_ratio"])
        boxes = MO.inst_rois(inp["roi_center"], inp["scale"])
        masks = [MO.paste_masks(MO.get_out_mask(o[k], "L1")[:, 0], boxes, (H, W), thr).cpu().numpy()
                 for k in ("mask", "full_mask")]
        if cfg.TEST.USE_PNP:
            pose = pnp_ransac_from_maps(o["coor_x"], o["coor_y"], o["coor_z"], o["mask"], inp["roi_coord_2d"], inp["im_H"],
                                        inp["im_W"], inp["roi_extent"], inp["roi_cam"], mask_thr=thr)
        else:
            pose = torch.cat([o["rot"], o["trans"][:, :, None]], 2)
        pose = pose.cpu().numpy()
        sid, iid = ts.images[idx]
        out[f"{sid}/{iid}"] = [G.save_record(a, pose[k], MO.encode(masks[0][k]), MO.encode(masks[1][k]), cfg.TEST.USE_PNP)
                               for k, a in enumerate(anns)]
    return out


def _same(a, b, poses_bitwise=True):
    assert list(a) == list(b)
    for k in a:
        assert len(a[k]) == len(b[k])
        for x, y in zip(a[k], b[k]):
            assert x["obj_id"] == y["obj_id"] and x["score"] == y["score"]
            assert x["bbox_est"].dtype == y["bbox_est"].dtype == np.float32 and np.array_equal(x["bbox_est"], y["bbox_est"])
            assert x["mask"] == y["mask"] and x["full_mask"] == y["full_mask"]
            assert x["R"].dtype == y["R"].dtype and x["t"].dtype == y["t"].dtype
            if poses_bitwise:
                assert np.array_equal(x["R"], y["R"]) and np.array_equal(x["t"], y["t"])


@pytest.mark.gpu
@pytest.mark.parametrize("use_pnp", [False, True])
def test_save_loop_matches_per_image_driver(dev, tmp_path, use_pnp):
    root, det = _tree(tmp_path, num_images=10, seed=8)
    cfg = _cfg(det, USE_PNP=use_pnp, PNP_TYPE="net_iter_pnp", USE_DEPTH_REFINE=True)   # neither applies on this path
    cfg.MODEL.POSE_NET.GEO_HEAD.MASK_THR_TEST = 0.5
    model = _model(cfg, dev)
    ts = G.TestSet(cfg, root)
    a = G.gdrn_save_result_of_dataset(cfg, model, root, str(tmp_path / "out64"), max_batch=64, test_set=ts)
    b = G.gdrn_save_result_of_dataset(cfg, model, root, str(tmp_path / "out1"), max_batch=1, test_set=ts)
    # bf16x3: network poses bitwise across batch sizes; RANSAC draws its hypotheses per ROI position in the batch
    _same(a, b, poses_bitwise=not use_pnp)
    ref = _per_image_driver(cfg, model, ts, dev)
    _same(b, ref, poses_bitwise=use_pnp)                          # one image per forward, as the driver runs them
    _same(a, ref, poses_bitwise=False)
    for k in a:
        for x, y in zip(b[k], ref[k]):
            assert np.abs(x["t"] - y["t"]).max() < 1e-3 and np.abs(x["R"] - y["R"]).max() < 1e-3
    assert sum(len(v) for v in a.values()) > 30
    assert sum(r["mask"]["counts"] != MO.encode(np.zeros((480, 640)))["counts"] for v in a.values() for r in v) > 5
    with open(tmp_path / "out64" / "results.pkl", "rb") as f:
        loaded = pickle.load(f)
    _same(loaded, a)


@pytest.mark.gpu
def test_save_loop_per_object(dev, tmp_path):
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    root, det = _tree(tmp_path, num_images=6, seed=6, dets_per_image=21)
    cfg = _cfg(det)
    g = cfg.MODEL.POSE_NET.GEO_HEAD
    g.XYZ_CLASS_AWARE = g.MASK_CLASS_AWARE = g.REGION_CLASS_AWARE = False
    cfg.MODEL.POSE_NET.NUM_CLASSES = 1
    objs = [2, 5, 11]
    sds = {o: make_state_dict(num_classes=1, seed=40 + o) for o in objs}
    ts = G.TestSet(cfg, root, objs)
    both = G.gdrn_save_result_of_dataset(cfg, G.build_model(cfg, sds, obj_ids=ts.obj_ids), root, str(tmp_path / "po"),
                                         train_obj_ids=objs)
    for o in objs:
        one = G.gdrn_save_result_of_dataset(cfg, G.build_model(cfg, sds[o]), root, str(tmp_path / f"o{o}"),
                                            train_obj_ids=[o])
        sub = {k: [r for r in v if r["obj_id"] == o] for k, v in both.items()}
        _same({k: v for k, v in sub.items() if v}, one, poses_bitwise=False)
    assert sum(len(v) for v in both.values()) == 6 * len(objs)


@pytest.mark.gpu
def test_cli_and_mask_tools(dev, tmp_path, capsys):
    from gdrnpp_bop2022_b200 import main_gdrn, mask_metrics
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    root, det = _tree(tmp_path, num_images=8, seed=9, dets_per_image=8)
    ckpt = str(tmp_path / "model_final.pth")
    torch.save({"model": make_state_dict(num_classes=21, seed=0)}, ckpt)
    conf = tmp_path / "cfg.py"
    conf.write_text(f"""
OUTPUT_DIR = {str(tmp_path / 'output')!r}
MODEL = dict(POSE_NET=dict(NAME="GDRN_double_mask", NUM_CLASSES=21, OUTPUT_RES=64,
                           BACKBONE=dict(INIT_CFG=dict(type="timm/convnext_base")),
                           GEO_HEAD=dict(NUM_REGIONS=64, XYZ_CLASS_AWARE=True, MASK_CLASS_AWARE=True, REGION_CLASS_AWARE=True,
                                         MASK_THR_TEST=0.5),
                           PNP_NET=dict(ROT_TYPE="allo_rot6d", TRANS_TYPE="centroid_z", Z_TYPE="REL", WITH_2D_COORD=True,
                                        REGION_ATTENTION=True),
                           LOSS_CFG=dict(MASK_LOSS_TYPE="L1", FULL_MASK_LOSS_TYPE="BCE")))
DATASETS = dict(TEST=("ycbv_bop_test",), DET_FILES_TEST=({det!r},), DET_THR=0.0, DET_TOPK_PER_OBJ=100)
VAL = dict(DATASET_NAME="ycbv", SPLIT="test", SPLIT_TYPE="", TARGETS_FILENAME="test_targets_bop19.json", USE_BOP=True)
TEST = dict(USE_PNP=False, SAVE_RESULTS_ONLY=False)
INPUT = dict(WITH_DEPTH=False, DZI_PAD_SCALE=1.5, MIN_SIZE_TEST=480, MAX_SIZE_TEST=640)
""")
    res = main_gdrn.main(["--config-file", str(conf), "--eval-only", "--datasets_root", root,
                          "--opts", f"MODEL.WEIGHTS={ckpt}", "TEST.SAVE_RESULTS_ONLY=True"])
    path = os.path.join(str(tmp_path / "output"), "inference_model_final", "ycbv_bop_test", "results.pkl")
    assert res["results"] == path and os.path.exists(path)
    with pytest.raises(SystemExit, match="exactly one DATASETS.TEST"):
        main_gdrn.main(["--config-file", str(conf), "--datasets_root", root, "--opts", f"MODEL.WEIGHTS={ckpt}",
                        "TEST.SAVE_RESULTS_ONLY=True", "DATASETS.TEST=('a','b')"])
    with open(path, "rb") as f:
        result = pickle.load(f)
    ts = G.TestSet(main_gdrn.load_py_config(str(conf)), root)
    base = os.path.join(root, "BOP_DATASETS", "ycbv", "test")
    obj = max({r["obj_id"] for v in result.values() for r in v}, key=lambda o: sum(r["obj_id"] == o for v in result.values() for r in v))
    for mask_type, key, d in (("vis", "mask", "mask_visib"), ("full", "full_mask", "mask")):
        capsys.readouterr()
        got = mask_metrics.main(["--dataset", "ycbv_bop_test", "--obj_id", str(obj), "--res_path", path, "--mask_type", mask_type,
                                 "--datasets_root", root])
        text = capsys.readouterr().out
        mious, f1s, skipped = [], [], 0
        for sid, iid in ts.images:
            preds = result.get(f"{sid}/{iid}", [])
            ids = [r["obj_id"] for r in preds]
            if obj not in ids:
                mious.append(0.0)
                f1s.append(0.0)
                continue
            gt_ids = [g["obj_id"] for g in G.bop_eval.load_json(os.path.join(base, f"{sid:06d}", "scene_gt.json"))[str(iid)]]
            if obj not in gt_ids:
                skipped += 1
                continue
            import cv2

            gt = cv2.imread(os.path.join(base, f"{sid:06d}", d, f"{iid:06d}_{gt_ids.index(obj):06d}.png"), -1).astype(bool)
            pred = MO.decode(preds[ids.index(obj)][key])
            mious.append(MO.compute_mean_iou(pred, gt))
            f1s.append(MO.f1_binary(pred, gt))
        assert got["skipped"] == skipped and got["num_scores"] == len(mious)
        assert f"mIoU (%): {np.mean(mious) * 100:.2f}" in text
        assert f"mean F1 score (%): {np.mean(f1s) * 100:.2f}" in text
        assert got["miou"] == pytest.approx(np.mean(mious), abs=1e-12) and got["f1"] == pytest.approx(np.mean(f1s), abs=1e-12)
