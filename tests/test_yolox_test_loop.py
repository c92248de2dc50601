"""The YOLOX dataset test loop (yolox_evaluator.py, main_yolox.py), its letterbox kernel (csrc/yolox_letterbox.cu) and
COCO box AP on the GPU (coco_eval.py, csrc/coco_eval.cu) against the NumPy restatement of COCOeval."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import coco_eval_oracle as CO


def _gt(boxes, areas=None, images=None, cats=None, crowd=None):
    anns = []
    for k, b in enumerate(boxes):
        anns.append({"id": k + 1, "image_id": 0 if images is None else images[k], "category_id": 0 if cats is None else cats[k],
                     "bbox": list(map(float, b)), "area": float(b[2] * b[3]) if areas is None else float(areas[k]),
                     "iscrowd": 0 if crowd is None else crowd[k]})
    return {"images": sorted({a["image_id"] for a in anns} | {0}), "annotations": anns}


def _dt(boxes, scores, images=None, cats=None):
    return [{"image_id": 0 if images is None else images[k], "category_id": 0 if cats is None else cats[k],
             "bbox": list(map(float, b)), "score": float(s)} for k, (b, s) in enumerate(zip(boxes, scores))]


# ---------------------------------------------------------------------------------------------------- CPU: oracle
def test_oracle_single_match_iou_078():
    r = CO.evaluate_boxes(_gt([[0, 0, 100, 100]]), _dt([[0, 0, 100, 78]], [0.9]), 1)
    # IoU 0.78 clears .50 ... .75 (6 of 10 thresholds)
    assert r["stats"][0] == pytest.approx(0.6, abs=1e-12)
    assert r["stats"][1:3] == pytest.approx([1.0, 1.0], abs=1e-12)   # pr = 1 / (1 + eps)
    assert r["stats"][5] == pytest.approx(0.6, abs=1e-12)
    assert r["stats"][3] == -1 and r["stats"][4] == -1          # no small / medium GT


def test_oracle_false_positive_ahead_of_true_positive():
    r = CO.evaluate_boxes(_gt([[0, 0, 100, 100]]), _dt([[200, 200, 50, 50], [0, 0, 100, 100]], [0.9, 0.8]), 1)
    assert r["stats"][0] == pytest.approx(0.5, abs=1e-12)      # pr = [0, .5], envelope [.5, .5]
    assert r["stats"][8] == 1.0 and r["stats"][6] == 0.0         # AR@100 = 1, AR@1: the top detection is the FP


def test_oracle_category_without_gt():
    r = CO.evaluate_boxes(_gt([[0, 0, 100, 100]]), _dt([[0, 0, 100, 100], [5, 5, 10, 10]], [0.9, 0.5], cats=[0, 1]), 2)
    assert np.all(r["precision"][:, :, 1] == -1) and np.all(r["recall"][:, 1] == -1)
    assert r["stats"][0] == pytest.approx(1.0, abs=1e-12) and r["stats"][3] == -1


def test_oracle_match_to_out_of_range_gt_is_ignored():
    g = _gt([[0, 0, 100, 100], [300, 300, 20, 20]])
    d = _dt([[0, 0, 100, 100], [300, 300, 20, 20]], [0.9, 0.8])
    r = CO.evaluate_boxes(g, d, 1)
    assert r["stats"][3] == pytest.approx(1.0, abs=1e-12)   # small: the large match is ignored, not a false positive
    e = r["evaluator"].eval_imgs[1]       # category 0, area "small", image 0
    assert e["dtIgnore"][0].tolist() == [True, False] and e["gtIgnore"].tolist() == [0, 1]


@pytest.mark.parametrize("fp_first,ap", [(True, 0.5), (False, 1.0)])
def test_oracle_ties_keep_input_order(fp_first, ap):
    boxes = [[200, 200, 50, 50], [0, 0, 100, 100]]
    d = _dt(boxes if fp_first else boxes[::-1], [0.7, 0.7])
    assert CO.evaluate_boxes(_gt([[0, 0, 100, 100]]), d, 1)["stats"][0] == pytest.approx(ap, abs=1e-12)


@pytest.mark.parametrize("n_fp,recall", [(100, 0.0), (99, 1.0)])
def test_oracle_more_than_100_detections(n_fp, recall):
    boxes = [[500 + 3 * k, 500, 10, 10] for k in range(n_fp)] + [[0, 0, 100, 100]]
    scores = [0.9 - 1e-3 * k for k in range(n_fp)] + [0.1]
    r = CO.evaluate_boxes(_gt([[0, 0, 100, 100]]), _dt(boxes, scores), 1)
    assert len(r["evaluator"].eval_imgs[0]["dtIds"]) == 100
    assert r["stats"][8] == recall


# ---------------------------------------------------------------------------------------------------- CPU: config / files
BASE_CFG = '''
import os.path as osp
from omegaconf import OmegaConf
train = dict(output_dir=osp.abspath(__file__).replace("configs", "output", 1)[0:-3], init_checkpoint="")
DATASETS = dict(TRAIN=("",), TEST=("",))
DATASETS = OmegaConf.create(DATASETS)
model = L(YOLOX)(backbone=L(YOLOPAFPN)(depth=1.0, width=1.0), head=L(YOLOXHead)(num_classes=80))
val = dict(eval_cached=False)
test = dict(test_dataset_names=DATASETS.TEST, test_size=(640, 640), conf_thr=0.01, nms_thr=0.65, amp_test=False,
            half_test=True)
dataloader.test = [L(build_yolox_test_loader)(dataset=L(Base_DatasetFromList)(preproc=L(ValTransform)(legacy=False)))
                   for n in test.test_dataset_names]
dataloader.evaluator = [L(YOLOX_COCOEvaluator)(dataset_name=n, filter_scene=False) for n in test.test_dataset_names]
'''
DERIVED_CFG = '''
from .yolox_base import train, val, test, model, dataloader, DATASETS  # noqa
model.backbone.depth = 0.33
model.backbone.width = 0.25
model.head.num_classes = 21
DATASETS.TEST = ["ycbv_bop_test"]
test.test_dataset_names = DATASETS.TEST
test.augment = True
test.scales = (1, 0.75, 0.83, 1.12, 1.25)
test.conf_thr = 0.001
'''


def _write_cfg(tmp_path, extra="", base_extra=""):
    d = tmp_path / "configs" / "yolox"
    d.mkdir(parents=True, exist_ok=True)
    (d / "yolox_base.py").write_text(BASE_CFG + base_extra)
    (d / "yolox_small_ycbv.py").write_text(DERIVED_CFG + extra)
    return str(d / "yolox_small_ycbv.py")


def test_config_reader_test_loop_fields(tmp_path):
    from gdrnpp_bop2022_b200.yolox_evaluator import check_test_config, precision_of
    from gdrnpp_bop2022_b200.yolox_model import load_yolox_config

    path = _write_cfg(tmp_path)
    c = load_yolox_config(path)
    assert c.test_dataset_names == ("ycbv_bop_test",) and c.half_test and not c.amp_test
    assert c.output_dir == path.replace("configs", "output", 1)[:-3]
    check_test_config(c)
    assert precision_of(c) == "bf16" and precision_of(c, "bf16x3") == "bf16x3"
    c.half_test = False
    assert precision_of(c) == "bf16x3"


@pytest.mark.parametrize("extra,base_extra,word", [
    ("", "dataloader.evaluator = [L(YOLOX_COCOEvaluator)(dataset_name=n, filter_scene=True) for n in test.test_dataset_names]\n",
     "filter_scene"),
    ("val.eval_cached = True\n", "", "val.eval_cached"),
    ("dataloader.test = [L(build_yolox_test_loader)(dataset=L(Base_DatasetFromList)(preproc=L(ValTransform)(legacy=True)))]\n",
     "", "legacy"),
    ('DATASETS.TEST = ["ycbv_bop_test", "lmo_bop_test"]\ntest.test_dataset_names = DATASETS.TEST\n', "",
     "test.test_dataset_names")])
def test_config_rejections(tmp_path, extra, base_extra, word):
    from gdrnpp_bop2022_b200.yolox_evaluator import check_test_config
    from gdrnpp_bop2022_b200.yolox_model import load_yolox_config

    with pytest.raises(NotImplementedError, match=word.replace(".", r"\.")):
        check_test_config(load_yolox_config(_write_cfg(tmp_path, extra, base_extra)))


@pytest.mark.skipif(not os.environ.get("GDRN_REFERENCE_SRC"), reason="GDRN_REFERENCE_SRC not set")
def test_config_reader_shipped_configs():
    import glob

    from gdrnpp_bop2022_b200.yolox_evaluator import SPLITS, check_test_config
    from gdrnpp_bop2022_b200.yolox_model import load_yolox_config

    files = sorted(glob.glob(os.path.join(os.environ["GDRN_REFERENCE_SRC"], "configs", "yolox", "bop_pbr", "yolox_x_*.py")))
    assert len(files) == 10
    for f in files:
        c = load_yolox_config(f)
        check_test_config(c)
        assert c.half_test and not c.amp_test and not c.eval_cached and not c.legacy and not c.filter_scene
        assert c.output_dir == os.path.abspath(f).replace("configs", "output", 1)[:-3]
        assert c.num_classes == len(SPLITS[c.test_dataset_names[0]][4])


def test_cli_overrides():
    from types import SimpleNamespace

    from gdrnpp_bop2022_b200.main_yolox import apply_overrides

    cfg = SimpleNamespace(augment=True, conf_thr=0.001, test_size=(640, 640))
    cfg, ck = apply_overrides(cfg, ["train.init_checkpoint=out/model_final.pth", "test.augment=False",
                                    "test.test_size=(320,320)", "DATASETS.TEST=['lmo_bop_test']"])
    assert ck == "out/model_final.pth" and cfg.augment is False and cfg.test_size == (320, 320)
    assert cfg.test_dataset_names == ("lmo_bop_test",)
    with pytest.raises(SystemExit):
        apply_overrides(cfg, ["model.head.num_classes=3"])


def test_cli_documented_argument_order():
    from gdrnpp_bop2022_b200.main_yolox import parse_args

    a = parse_args(["--config-file", "configs/yolox/bop_pbr/cfg.py", "--eval-only", "--datasets_root", "datasets",
                    "train.init_checkpoint=CKPT", "test.augment=False", "--det_file", "out/dets.json"])
    assert a.det_file == "out/dets.json" and a.opts == ["train.init_checkpoint=CKPT", "test.augment=False"]
    a = parse_args(["--config-file", "c.py", "--det_file", "d.json", "train.init_checkpoint=CKPT", "test.scales=(1, 0.75)"])
    assert a.det_file == "d.json" and a.opts == ["train.init_checkpoint=CKPT", "test.scales=(1, 0.75)"]


def _mini_split(root, dataset, masks):
    """A BOP test split without images: scene 2, masks {im_id: [(obj_id, mask uint8 [8,8])]}, bbox_obj per instance."""
    import cv2

    sdir = os.path.join(root, "BOP_DATASETS", dataset, "test", "000002")
    os.makedirs(os.path.join(sdir, "mask_visib"))
    gt, info, targets = {}, {}, []
    for im_id, insts in masks.items():
        gt[str(im_id)] = [{"obj_id": o} for o, _ in insts]
        info[str(im_id)] = [{"bbox_obj": [k, 1, 3, 4]} for k in range(len(insts))]
        for k, (o, m) in enumerate(insts):
            cv2.imwrite(os.path.join(sdir, "mask_visib", f"{im_id:06d}_{k:06d}.png"), m)
            targets.append({"scene_id": 2, "im_id": im_id, "obj_id": o, "inst_count": 1})
    for name, c in (("scene_gt.json", gt), ("scene_gt_info.json", info)):
        json.dump(c, open(os.path.join(sdir, name), "w"))
    json.dump(targets, open(os.path.join(root, "BOP_DATASETS", dataset, "test_targets_bop19.json"), "w"))


@pytest.mark.parametrize("name,dataset", [("lmo_bop_test", "lmo"), ("ycbv_bop_test", "ycbv")])
def test_test_set_mask_rule_and_image_ids(tmp_path, name, dataset):
    """Only ycbv_bop_test's loader drops an instance whose mask_visib sums to < 3; LM-O's keeps it (COCO area 0).
    ycbv's image_id counts every image of the targets file, LM-O's is the BOP im_id."""
    from gdrnpp_bop2022_b200.yolox_evaluator import YoloxTestSet

    empty, full = np.zeros((8, 8), np.uint8), np.full((8, 8), 255, np.uint8)
    two_ones = np.zeros((8, 8), np.uint8)
    two_ones[0, :2] = 1                                          # 2 nonzero pixels, sum 2
    masks = {3: [(1, empty), (5, full)], 5: [(8, empty)], 9: [(9, two_ones), (1, full)]}
    root = str(tmp_path / "datasets")
    _mini_split(root, dataset, masks)
    ts = YoloxTestSet(name, root)
    anns = [(a["image_id"], a["category_id"], a["area"]) for a in ts.gt["annotations"]]
    lab = ts.obj_ids.index
    if dataset == "lmo":
        assert ts.images == [(2, 3), (2, 5), (2, 9)] and ts.image_ids == [3, 5, 9]
        assert anns == [(3, lab(1), 0), (3, lab(5), 64), (5, lab(8), 0), (9, lab(9), 2), (9, lab(1), 64)]
    else:
        assert ts.images == [(2, 3), (2, 9)] and ts.image_ids == [0, 2]   # image 5 dropped, its id skipped
        assert anns == [(0, lab(5), 64), (2, lab(1), 64)]
    assert ts.gt["images"] == ts.image_ids


def test_converted_file_lmo_labels_round_trip(tmp_path):
    from gdrnpp_bop2022_b200 import gdrn_evaluator as G
    from gdrnpp_bop2022_b200.yolox_evaluator import SPLITS, convert_det_to_ours, save_json

    obj_ids = SPLITS["lmo_bop_test"][4]
    bop = [{"scene_id": 2, "image_id": 3, "category_id": c, "score": 0.5 + 0.01 * c, "bbox": [1.5, 2.0, 30.25, 40.0],
            "time": 0.02} for c in range(1, 9)] + [{"scene_id": 2, "image_id": 7, "category_id": 2, "score": 0.3,
                                                      "bbox": [0.0, 0.0, 5.0, 5.0], "time": 0.01}]
    outs = convert_det_to_ours(bop, obj_ids)
    assert [d["obj_id"] for d in outs["2/3"]] == [1, 5, 6, 8, 9, 10, 11, 12]
    path = str(tmp_path / "dets.json")
    save_json(path, outs)
    text = open(path).read()
    assert text.startswith('{\n  "2/3": [{"bbox_est": [1.5, 2.0, 30.25, 40.0], "obj_id": 1,') and text.endswith("]\n}")
    loaded = G.load_detections(json.load(open(path)), [(2, 3), (2, 7)], G.DATASET_OBJ_IDS["lmo"], top_k_per_obj=100)
    assert [a["obj_id"] for a in loaded[0][1]] == [1, 5, 6, 8, 9, 10, 11, 12]
    assert [a["label"] for a in loaded[0][1]] == list(range(8)) and loaded[1][1][0]["obj_id"] == 5


# ---------------------------------------------------------------------------------------------------- GPU: letterbox
def _host_letterbox(img, test_size):
    """base_data_from_list.load_resized_img + ValTransform(legacy=False) with host cv2."""
    import cv2

    from gdrnpp_bop2022_b200.predictor_yolo import preproc

    r = min(test_size[0] / img.shape[0], test_size[1] / img.shape[1])
    img1 = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR).astype(np.uint8)
    return preproc(img1, test_size)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,C,N,test_size", [
    (480, 640, 3, 1, (640, 640)), (480, 640, 3, 7, (640, 640)), (540, 720, 3, 7, (640, 640)),
    (960, 1280, 1, 1, (640, 640)), (960, 1280, 1, 7, (640, 640)), (240, 320, 3, 7, (640, 640)),
    (20, 47, 3, 7, (64, 96)), (250, 333, 3, 1, (416, 416))])
def test_letterbox_bit_exact(dev, H, W, C, N, test_size):
    from gdrnpp_bop2022_b200.native_ops import letterbox_ratio, yolox_letterbox

    rng = np.random.RandomState(H + W + N)
    imgs = rng.randint(0, 256, (N, H, W, C)).astype(np.uint8)
    out = yolox_letterbox(torch.from_numpy(imgs).to(dev), test_size).cpu().numpy()
    for n in range(N):
        im3 = np.repeat(imgs[n], 3, axis=2) if C == 1 else imgs[n]     # read_image_mmcv(..., "BGR") of a gray image
        assert np.array_equal(out[n], _host_letterbox(im3, test_size)), n
    _, (h1, w1) = letterbox_ratio(H, W, test_size)
    twice = letterbox_ratio(h1, w1, test_size)[1] != (h1, w1)
    print(f"{W}x{H} C={C} -> {w1}x{h1}, second resize {'applied' if twice else 'identity'}")
    if (H, W) == (20, 47):
        assert twice


# ---------------------------------------------------------------------------------------------------- GPU: coco_eval
def _random_set(seed, n_img=320, K=5):
    rng = np.random.RandomState(seed)
    anns, dets = [], []
    for i in range(n_img):
        if i % 17 == 5:
            continue                                   # an image with neither GT nor detections
        for _ in range(rng.randint(0, 5)):
            side = rng.choice([rng.uniform(5, 200), rng.choice([32.0, 96.0]) + rng.uniform(-1, 1)])
            w, h = side, side * rng.uniform(0.8, 1.25)
            x, y = rng.uniform(0, 500, 2)
            c = int(rng.randint(K))
            area = w * h if rng.rand() < 0.5 else float(rng.choice([32 ** 2, 96 ** 2, rng.uniform(500, 12000)]))
            anns.append({"image_id": i, "category_id": c, "bbox": [x, y, w, h], "area": area,
                         "iscrowd": int(rng.rand() < 0.05)})
            for _ in range(rng.randint(0, 4)):        # detections around the GT
                j = rng.normal(0, 0.15 * w, 4)
                dets.append({"image_id": i, "category_id": c if rng.rand() < 0.9 else int(rng.randint(K)),
                             "bbox": [x + j[0], y + j[1], max(w + j[2], 1.0), max(h + j[3], 1.0)],
                             "score": float(np.round(rng.uniform(0, 1), 2))})   # rounded: many ties
        for _ in range(rng.randint(0, 3) if i % 7 else 120):   # background detections; some images over 100
            s = rng.uniform(4, 150)
            dets.append({"image_id": i, "category_id": int(rng.randint(K)), "bbox": [*rng.uniform(0, 500, 2), s, s * 0.9],
                         "score": float(np.round(rng.uniform(0, 1), 2))})
    images = [i for i in range(n_img) if i % 17 != 5 or i % 34 == 5]   # a few empty images stay in the GT image list
    return {"images": images, "annotations": anns}, dets, K


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_coco_eval_matches_oracle(dev, seed):
    from gdrnpp_bop2022_b200.coco_eval import evaluate_boxes

    gt, dets, K = _random_set(seed)
    ref = CO.evaluate_boxes(gt, dets, K)
    got = evaluate_boxes(gt, dets, K, device=dev, return_matches=True)
    ev, m = ref["evaluator"], got["matches"]
    I, A = len(ev.img_ids), len(CO.AREA_RNG)
    n_pairs = 0
    for p, (img, cat) in enumerate(m["pairs"]):
        g0, g1 = m["pair_gt_off"][p], m["pair_gt_off"][p + 1]
        k0, k1 = m["pair_kept_off"][p], m["pair_kept_off"][p + 1]
        for a in range(A):
            e = ev.eval_imgs[cat * A * I + a * I + ev.img_ids.index(img)]
            gig = m["gt_ignore"][a, g0:g1]
            perm = np.argsort(gig, kind="mergesort")          # evaluateImg's GT order: ignored last
            assert e["dtIds"] == m["kept_det_id"][k0:k1].tolist()
            assert e["gtIds"] == m["gt_id"][g0:g1][perm].tolist()
            assert np.array_equal(e["gtIgnore"], gig[perm])
            assert np.array_equal(e["dtMatches"], m["dt_match"][a, :, k0:k1])
            assert np.array_equal(e["dtIgnore"], m["dt_ignore"][a, :, k0:k1].astype(bool))
            assert np.array_equal(e["gtMatches"], m["gt_match"][a][:, g0:g1][:, perm])
        n_pairs += 1
    assert n_pairs == sum(e is not None for e in ev.eval_imgs) // A
    assert np.abs(got["precision"] - ref["precision"]).max() <= 1e-12
    assert np.abs(got["recall"] - ref["recall"]).max() <= 1e-12
    assert np.allclose(got["stats"], ref["stats"], rtol=0, atol=1e-12)
    for k in range(K):
        pk = ref["precision"][:, :, k, 0, -1]
        want = np.mean(pk[pk > -1]) * 100 if (pk > -1).any() else float("nan")
        assert got[f"AP-obj_{k + 1:06d}"] == pytest.approx(want, abs=1e-10, nan_ok=True)
    print("stats", np.round(got["stats"], 4).tolist())


# ---------------------------------------------------------------------------------------------------- GPU: the loop
TEST_SIZE = (256, 320)


def _split(tmp_path, num_images=14, seed=3, **kw):
    """A synthetic ycbv_bop_test split with mask_visib: rectangle masks over each instance's bbox_obj, cut to the image;
    every fifth instance and every instance of the third image have empty masks (instance / image dropped)."""
    import cv2

    from gdrnpp_bop2022_b200.synthetic import write_bop_tree

    root = str(tmp_path / "datasets")
    write_bop_tree(root, num_images=num_images, seed=seed, **kw)
    split = os.path.join(root, "BOP_DATASETS", "ycbv", "test")
    n = 0
    for scene in sorted(os.listdir(split)):
        sdir = os.path.join(split, scene)
        if not scene.isdigit():
            continue
        info = json.load(open(os.path.join(sdir, "scene_gt_info.json")))
        os.makedirs(os.path.join(sdir, "mask_visib"), exist_ok=True)
        for im_id, insts in sorted(info.items(), key=lambda p: int(p[0])):
            H, W = cv2.imread(os.path.join(sdir, "rgb", f"{int(im_id):06d}.png")).shape[:2]
            for k, g in enumerate(insts):
                m = np.zeros((H, W), np.uint8)
                x, y, w, h = g["bbox_obj"]
                if k % 5 != 4 and n != 2:
                    m[max(y, 0):max(min(y + h, H), 0), max(x, 0):max(min(x + w, W), 0)] = 255
                cv2.imwrite(os.path.join(sdir, "mask_visib", f"{int(im_id):06d}_{k:06d}.png"), m)
            n += 1
    return root


def _yolox(dev, precision, max_batch=8, seed=0):
    from gdrnpp_bop2022_b200.synthetic import make_yolox_state_dict
    from gdrnpp_bop2022_b200.yolox_model import YOLOX
    from oracle.yolox_oracle import yolox_forward

    sd = make_yolox_state_dict(yolox_forward, 0.33, 0.25, 21, seed=seed, calib_hw=TEST_SIZE, calib_batch=2, device=dev)
    m = YOLOX(0.33, 0.25, 21, max_batch=max_batch, precision=precision).eval()
    m.load_state_dict(sd)
    return m.to(dev), sd


def _cfg(augment):
    from types import SimpleNamespace

    return SimpleNamespace(test_size=TEST_SIZE, conf_thr=0.01, nms_thr=0.65, augment=augment,
                           scales=(1, 0.75, 0.83, 1.12, 1.25) if augment else None, num_classes=21,
                           test_dataset_names=("ycbv_bop_test",), half_test=False, amp_test=False)


def _driver_rows(cfg, model, ts, dev):
    """One image at a time as the reference does: host cv2 pre-processing, model(x), postprocess, float32 CPU box math."""
    from gdrnpp_bop2022_b200.gdrn_evaluator import read_image
    from gdrnpp_bop2022_b200.yolox_post import postprocess

    coco, bop = [], []
    for idx, ((sid, iid), path) in enumerate(zip(ts.images, ts.paths)):
        im = read_image(path)
        im = np.repeat(im, 3, axis=2) if im.shape[2] == 1 else im
        x = torch.from_numpy(_host_letterbox(im, cfg.test_size))[None].to(dev)
        kw = {"augment": True, "cfg": cfg} if cfg.augment else {}
        out = postprocess(model(x, **kw)["det_preds"], 21, cfg.conf_thr, cfg.nms_thr)[0]
        if out is None:
            continue
        det = out.cpu()
        bboxes = det[:, 0:4]
        scale = min(cfg.test_size[0] / float(im.shape[0]), cfg.test_size[1] / float(im.shape[1]))
        bboxes /= scale
        bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 0]
        bboxes[:, 3] = bboxes[:, 3] - bboxes[:, 1]
        labels, scores = det[:, 6], det[:, 4] * det[:, 5]
        for i in range(bboxes.shape[0]):
            coco.append({"image_id": ts.image_ids[idx], "category_id": int(labels[i]), "score": scores[i].numpy().item(),
                         "bbox": bboxes[i].numpy().tolist()})
            bop.append({"scene_id": sid, "image_id": iid, "category_id": int(labels[i]) + 1,
                        "score": scores[i].numpy().item(), "bbox": bboxes[i].numpy().tolist()})
    return coco, bop


def _loop_files(cfg, model, root, ts, out_dir, max_batch):
    from gdrnpp_bop2022_b200 import yolox_evaluator as YE

    rec = YE.yolox_inference_on_dataset(cfg, model, root, max_batch=max_batch, test_set=ts)
    res = YE.YoloxDatasetEvaluator(cfg, ts, out_dir, config_name="small").evaluate(rec)
    load = lambda k: json.load(open(res["files"][k]))
    return load("coco"), load("bop"), load("det_file"), res


def _strip_time(rows):
    return [{k: v for k, v in r.items() if k != "time"} for r in rows]


def _close(a, b, px, score):
    assert [(r["image_id"], r["category_id"]) for r in a] == [(r["image_id"], r["category_id"]) for r in b]
    eb = max((abs(x - y) for r, s in zip(a, b) for x, y in zip(r["bbox"], s["bbox"])), default=0.0)
    es = max((abs(r["score"] - s["score"]) for r, s in zip(a, b)), default=0.0)
    assert eb < px and es < score, (eb, es)
    return eb, es


@pytest.mark.gpu
@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_loop_matches_per_image_driver(dev, tmp_path, precision, augment):
    from gdrnpp_bop2022_b200 import yolox_evaluator as YE

    root = _split(tmp_path)
    ts = YE.YoloxTestSet("ycbv_bop_test", root)
    assert 0 < len(ts.images) < 14                                   # the image without kept instances is dropped
    cfg = _cfg(augment)
    model, _ = _yolox(dev, precision)
    c8, b8, d8, res = _loop_files(cfg, model, root, ts, str(tmp_path / "b8"), 8)
    c1, b1, d1, _ = _loop_files(cfg, model, root, ts, str(tmp_path / "b1"), 1)
    coco, bop = _driver_rows(cfg, model, ts, dev)
    assert len(c8) > 20 and "bbox" in res and np.isfinite(res["bbox"]["AP50"])
    assert [r["time"] for r in b8] and all(r["time"] > 0 for r in b8)
    if precision == "bf16x3":
        assert c8 == c1 and _strip_time(b8) == _strip_time(b1)      # bitwise: k-order does not depend on B
        assert c8 == coco and _strip_time(b8) == bop
    else:
        _close(c8, c1, 2.0, 2e-2)
        print("bf16 loop vs driver:", _close(c8, coco, 2.0, 2e-2))
    keys = sorted({f"{r['scene_id']}/{r['image_id']}" for r in b8}, key=lambda s: tuple(map(int, s.split("/"))))
    assert list(d8) == keys and sum(len(v) for v in d8.values()) == len(b8)


@pytest.mark.gpu
def test_main_yolox_feeds_main_gdrn(dev, tmp_path):
    from gdrnpp_bop2022_b200 import gdrn_evaluator as G
    from gdrnpp_bop2022_b200 import main_yolox

    root = _split(tmp_path, num_images=6, seed=8)
    cfg_path = _write_cfg(tmp_path, "test.test_size = (256, 320)\ntest.conf_thr = 0.3\n")
    _, sd = _yolox(dev, "bf16x3")
    ckpt = str(tmp_path / "yolox.pth")
    torch.save({"model": sd}, ckpt)
    det_file = str(tmp_path / "test_bboxes" / "yolox_small_ycbv_bop_test.json")
    res = main_yolox.main(["--config-file", cfg_path, "--eval-only", "--datasets_root", root, "--det_file", det_file,
                           f"train.init_checkpoint={ckpt}", f"train.output_dir={tmp_path / 'out'}", "test.augment=False"])
    assert os.path.exists(res["files"]["bop"]) and res["files"]["det_file"] == det_file
    from test_test_loop import _cfg as gdrn_cfg
    from test_test_loop import _model

    cfg = gdrn_cfg(det_file)
    cfg.DATASETS.DET_TOPK_PER_OBJ = 1
    model = _model(cfg, dev)
    rows = G.gdrn_inference_on_dataset(cfg, model, root)
    assert rows
    cfg.VAL.SAVE_BOP_CSV_ONLY = True
    out = G.GdrnDatasetEvaluator(cfg, root, str(tmp_path / "pose"), "cfg_test").evaluate(rows)
    assert os.path.getsize(out["csv"]) > 0
