"""The YOLOX training batcher (gdrnpp_bop2022_b200/yolox_train_batch.py, csrc/yolox_train_aug.cu) against the NumPy /
cv2 restatement in oracle/yolox_train_batch_oracle.py: records and host box arithmetic on the CPU, every kernel and
whole batches bit for bit on the GPU."""
import numpy as np
import pytest

from gdrnpp_bop2022_b200 import synthetic
from gdrnpp_bop2022_b200 import yolox_train_batch as YT
from gdrnpp_bop2022_b200.yolox_model import load_yolox_config
from oracle import yolox_train_batch_oracle as YO


@pytest.fixture(scope="module")
def lmo(tmp_path_factory):
    root = tmp_path_factory.mktemp("yolox_train")
    synthetic.write_bop_train_tree(str(root), dataset="lmo", num_images=12, obj_ids=(1, 5, 6, 2), insts_per_image=4)
    cfg = load_yolox_config(synthetic.write_yolox_train_config(str(root / "configs")))
    return str(root), cfg


@pytest.fixture(scope="module")
def tless(tmp_path_factory):
    """Two image sizes, both resized by load_resized_img: 720x540 PBR and 400x400 primesense."""
    root = tmp_path_factory.mktemp("yolox_train_tless")
    synthetic.write_bop_train_tree(str(root), dataset="tless", num_images=6, H=540, W=720, obj_ids=(1, 2, 3))
    synthetic.write_bop_train_tree(str(root), dataset="tless", num_images=6, H=400, W=400, obj_ids=(1, 2, 3), seed=1,
                                   split="train_primesense")
    path = synthetic.write_yolox_train_config(str(root / "configs"), train=("tless_pbr_train", "tless_primesense_train"),
                                              test="tless_bop_test_primesense")
    return str(root), load_yolox_config(path)


def _with(cfg, **wrap):
    import copy

    c = copy.deepcopy(cfg)
    c.aug_wrapper.update(wrap)
    return c


def _decode(ts, rec):
    return YT.decode(ts, rec, range(len(rec["mosaic"])))


def _labels(ts):
    return lambda i: ts.images[i]["labels"]


# --------------------------------------------------------------------------------------------- CPU
def test_config_reads_the_training_loader(lmo):
    _, cfg = lmo
    assert cfg.train_img_size == (640, 640) and cfg.train_dataset_names == ("lmo_pbr_train",)
    assert cfg.train_total_batch_size == 32 and cfg.no_aug_epochs == 15
    w = cfg.aug_wrapper
    assert (w["mosaic_scale"], w["degrees"], w["shear"], w["mixup_prob"], w["preproc.max_labels"]) == ((0.1, 2), 10.0, 2.0,
                                                                                                       1.0, 120)
    assert (w["HSV_H"], w["HSV_S"], w["HSV_V"], w["FORMAT"], w["COLOR_AUG_TYPE"]) == (0.015, 0.7, 0.4, "RGB", "code")


def test_train_set_follows_the_registrar(lmo):
    root, cfg = lmo
    ts = YT.YoloxTrainSet(cfg, root)
    assert ts.obj_ids == [1, 5, 6, 8, 9, 10, 11, 12]
    for im in ts.images:
        lab = im["labels"]
        assert set(lab[:, 4].astype(int)) <= {0, 1, 2} and (lab[:, 2] > lab[:, 0]).all() and (lab[:, 3] > lab[:, 1]).all()
        assert lab[:, [0, 2]].max(initial=0) <= 640 and lab[:, [1, 3]].max(initial=0) <= 480


def test_records_are_deterministic(lmo):
    root, cfg = lmo
    ts = YT.YoloxTrainSet(cfg, root)
    s = YT.Sampler(cfg, ts)
    a = s.draw(np.random.default_rng([0, 2000]), 16)
    b = s.draw(np.random.default_rng([0, 2000]), 16)
    c = s.draw(np.random.default_rng([0, 2001]), 16)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert not np.array_equal(a["index"], c["index"])


def test_host_boxes_match_the_oracle(lmo):
    """Mosaic with and without mixup, with and without its flip, non-mosaic samples, the min(w, h) > 1 fallback and a
    sample with more than 120 boxes."""
    root, cfg = lmo
    ts = YT.YoloxTrainSet(cfg, root)
    ts.images[0]["labels"] = np.array([[10.0, 10.0, 10.5, 200.0, 1.0]])   # w < 1 everywhere: the fallback
    many = np.tile(ts.images[1]["labels"][:1], (130, 1))
    many[:, :4] += np.arange(130)[:, None] * 0.5
    ts.images[1]["labels"] = many
    s = YT.Sampler(_with(cfg, mosaic_prob=0.5, COLOR_AUG_PROB=0.0), ts)
    rec = s.draw(np.random.default_rng(7), 64)
    flip = rec["mixup_flip"].astype(bool)
    mix, mos = rec["mixup"].astype(bool), rec["mosaic"].astype(bool)
    assert (mix & flip).any() and (mix & ~flip).any() and (~mos).any()
    assert rec["fallback"][~mos].any()
    assert (rec["targets"][:, -1, 3] > 0).any(), "no sample fills all 120 rows"
    _, targets = YO.replay(rec, _decode(ts, rec), _labels(ts), source_format="RGB")
    np.testing.assert_allclose(rec["targets"], targets, rtol=0, atol=1e-9)


def _shrink_visible_masks(split_dir, counts):
    """Rewrite instance 0 and 2 of every image to a visible mask of a few pixels (a block at (50, 50)), with its
    scene_gt_info px_count_visib and bbox_visib to match."""
    import json
    import math
    import os

    import cv2

    j = 0
    for scene in sorted(d for d in os.listdir(split_dir) if d.isdigit()):
        sdir = os.path.join(split_dir, scene)
        with open(os.path.join(sdir, "scene_gt_info.json")) as f:
            info = json.load(f)
        for im_id in info:
            for k in (0, 2):
                n = counts[j % len(counts)]
                j += 1
                path = os.path.join(sdir, "mask_visib", "{:06d}_{:06d}.png".format(int(im_id), k))
                m = cv2.imread(path, cv2.IMREAD_UNCHANGED)
                m[:] = 0
                side = max(1, math.ceil(math.sqrt(n)))
                for i in range(n):
                    m[50 + i // side, 50 + i % side] = 255
                cv2.imwrite(path, m)
                info[im_id][k]["px_count_visib"] = n
                info[im_id][k]["bbox_visib"] = [50, 50, min(n, side), math.ceil(n / side)] if n else [-1, -1, -1, -1]
        with open(os.path.join(sdir, "scene_gt_info.json"), "w") as f:
            json.dump(info, f)


@pytest.mark.parametrize("name", sorted(YT.TRAIN_SPLITS))
def test_train_set_area_rule_matches_the_registrar(tmp_path, monkeypatch, name):
    """Instances of 0-65 visible pixels against the registrars' own rule on the mask PNG: `area < 30` / `<= 64` on the
    pixel count where the registrar casts the mask to bool, on 255 x the count where it sums the raw PNG."""
    from gdrnpp_bop2022_b200.yolox_evaluator import SPLITS

    sp = YT.TRAIN_SPLITS[name]
    synthetic.write_bop_train_tree(str(tmp_path), dataset=sp.dataset, num_images=8, H=sp.hw[0], W=sp.hw[1],
                                   obj_ids=(1, 5) if sp.dataset == "lmo" else (1, 2), split=sp.split)
    _shrink_visible_masks(str(tmp_path / "BOP_DATASETS" / sp.dataset / sp.split), [0, 1, 4, 20, 29, 30, 64, 65])
    cfg = load_yolox_config(synthetic.write_yolox_train_config(str(tmp_path / "configs"), train=(name,),
                                                               test=YT.LABEL_SPLIT[sp.dataset]))
    ts = YT.YoloxTrainSet(cfg, str(tmp_path))
    ref = YO.registrar_images(str(tmp_path), name, list(SPLITS[YT.LABEL_SPLIT[sp.dataset]].obj_ids))
    assert [im["path"] for im in ts.images] == [p for p, _ in ref]
    for im, (_, lab) in zip(ts.images, ref):
        assert np.array_equal(im["labels"], lab)
    # the other kind of rule gives other samples on these masks, so the comparison above tells the two apart
    monkeypatch.setitem(YT.TRAIN_SPLITS, name, sp._replace(mask_value=256 - sp.mask_value))
    other = YT.YoloxTrainSet(cfg, str(tmp_path))
    assert sum(len(im["labels"]) for im in other.images) != sum(len(lab) for _, lab in ref)


@pytest.mark.parametrize("setting, value", [
    ("COLOR_AUG_TYPE", "ROI10D"), ("COLOR_AUG_CODE", "Sequential([Sometimes(0.5, Fliplr(0.5))])"),
    ("mosaic_prob", 1.5), ("mixup_prob", -0.1)])
def test_rejections_name_the_setting(lmo, setting, value):
    root, cfg = lmo
    with pytest.raises(Exception, match=setting if setting != "COLOR_AUG_CODE" else "Fliplr"):
        YT.YoloxTrainSet(_with(cfg, **{setting: value}), root)


def test_rejects_image_size_and_datasets(lmo):
    root, cfg = lmo
    import copy

    c = copy.deepcopy(cfg)
    c.train_img_size = (416, 416)
    with pytest.raises(NotImplementedError, match="img_size"):
        YT.YoloxTrainSet(c, root)
    for name in ("ycbv_train_real", "lm_pbr_13_train"):
        c = copy.deepcopy(cfg)
        c.train_dataset_names = (name,)
        with pytest.raises(NotImplementedError, match=name):
            YT.YoloxTrainSet(c, root)


# --------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["BGR", "RGB"])
def test_hsv_kernel_matches_cv2_over_all_colours(lib, dev, fmt):
    import torch

    from gdrnpp_bop2022_b200 import _lib

    allc = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(allc >> 16) & 255, (allc >> 8) & 255, allc & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    # hue wrap-around (r0 > 1), saturation / value clipping (r > 1), shrinking gains, and the identity
    for gains in ([1.5, 1.5, 1.5], [0.5, 0.5, 0.5], [1.0149, 1.69, 0.61], [0.985, 0.31, 1.39], [1.0, 1.0, 1.0]):
        d = torch.from_numpy(img.copy()).to(dev)
        ent = torch.tensor([[0, img.shape[0] * img.shape[1]]], dtype=torch.int64, device=dev)
        lut = torch.from_numpy(YT.hsv_luts(np.array(gains))[None].copy()).to(dev)
        _lib.check(lib.yolox_train_hsv(_lib.ptr(d), _lib.ptr(ent), _lib.ptr(lut), 1, img.shape[0] * img.shape[1],
                                       int(fmt == "RGB"), _lib.current_stream()), "yolox_train_hsv")
        ref = img.copy()
        YO.augment_hsv(ref, np.array(gains), fmt)
        got = d.cpu().numpy()
        assert np.array_equal(got, ref), f"gains {gains}: {(got != ref).any(-1).sum()} pixels differ"


def _crafted(s, rng, n, **fields):
    rec = s.draw(rng, n)
    for k, v in fields.items():
        rec[k][:] = v
    return rec


@pytest.mark.gpu
def test_mosaic_affine_matches_the_oracle(lib, dev, lmo):
    import torch

    root, cfg = lmo
    ts = YT.YoloxTrainSet(cfg, root)
    s = YT.Sampler(_with(cfg, enable_mixup=False, COLOR_AUG_PROB=0.0, AUG_HSV_PROB=0.0), ts)
    rec = _crafted(s, np.random.default_rng(3), 12, t_on=0, w_hsv=0)
    # the four centre quadrants and their extremes, extreme angles / scales / shears, tiles fully outside the output
    rec["center"][:] = [(320, 320), (959, 320), (320, 959), (959, 959), (640, 640), (321, 958), (700, 400), (500, 900),
                        (640, 640), (640, 640), (400, 800), (900, 350)]
    rec["affine"][:] = [(0, 1, 0, 0, 0, 0), (10, 0.1, 2, -2, 0.1, -0.1), (-10, 2, -2, 2, -0.1, 0.1), (179, 1.3, 0, 0, 0, 0),
                        (45, 0.5, 30, -30, 0.5, 0.5), (-90, 1.7, 1, 1, -0.3, 0.2), (0, 0.1, 0, 0, 0.9, 0.9),
                        (5, 2, 0, 0, -1.5, -1.5), (0, 1, 0, 0, 0.5, 0), (0, 0.5, 0, 0, -0.5, 0.2), (-170, 0.9, 15, 5, 0, 0),
                        (90, 1, -45, 0, 0.05, -0.05)]
    images = _decode(ts, rec)
    _, st = YT.build_images(s, rec, images, dev)
    plane = 640 * 640 * 3
    got = st["pool"][:12 * plane].view(12, 640, 640, 3).cpu().numpy()
    for b in range(12):
        ref, _ = YO.mosaic(rec, b, images[b], _labels(ts), (640, 640))
        assert np.array_equal(got[b], ref), f"sample {b}: {(got[b] != ref).any(-1).sum()} pixels differ"
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_mixup_matches_the_oracle(lib, dev, lmo):
    root, cfg = lmo
    ts = YT.YoloxTrainSet(cfg, root)
    s = YT.Sampler(_with(cfg, mixup_prob=1.0, COLOR_AUG_PROB=0.0, AUG_HSV_PROB=0.0), ts)
    rec = _crafted(s, np.random.default_rng(5), 8, t_on=0, w_hsv=0, mosaic=1, mixup=1)
    rec["cp_index"][:] = np.nonzero(ts.with_labels)[0][0]
    jits = [0.5, 0.5004, 0.77, 0.999, 1.0, 1.23, 1.5, 1.4999]
    for b, jit in enumerate(jits):
        rec["jit"][b], rec["mixup_flip"][b] = jit, b % 2
        extra = max(int(640 * jit), 640) - 640
        rec["offset"][b] = (0, 0) if extra == 0 else ((extra - 1, 0) if b % 4 < 2 else (0, extra - 1))
    images = _decode(ts, rec)
    _, st = YT.build_images(s, rec, images, dev)
    got = st["pool"][:8 * 640 * 640 * 3].view(8, 640, 640, 3).cpu().numpy()
    for b in range(8):
        img, boxes = YO.mosaic(rec, b, images[b], _labels(ts), (640, 640))
        ref, _ = YO.mixup(rec, b, img, boxes, images[b][4], ts.images[int(rec["cp_index"][b])]["labels"], (640, 640))
        assert np.array_equal(got[b], ref), f"jit {jits[b]}: {(got[b] != ref).any(-1).sum()} pixels differ"


def _check_batch(batcher, ts, fmt):
    imgs, targets, img_info, img_id = next(batcher)
    rec = batcher.last_records
    ref_imgs, ref_t = YO.replay(rec, _decode(ts, rec), _labels(ts), source_format=fmt)
    got = imgs.cpu().numpy()
    bad = [b for b in range(len(got)) if not np.array_equal(got[b], ref_imgs[b])]
    assert not bad, f"samples {bad} differ ({[(got[b] != ref_imgs[b]).sum() for b in bad]} values)"
    np.testing.assert_allclose(targets.cpu().numpy(), ref_t, rtol=0, atol=1e-6)
    assert imgs.shape == (len(got), 3, 640, 640) and targets.shape == (len(got), 120, 5)
    assert img_info[0].shape == (len(got),) and img_id.shape == (len(got), 1)
    # a mosaic sample: (mix_img.shape[1], mix_img.shape[0]) of its CHW image and the image id of its last tile;
    # otherwise its registrar's (height, width) and its own image id
    for b in range(len(got)):
        if rec["mosaic"][b]:
            want = (640, 3, ts.images[int(rec["index"][b, 3])]["image_id"])
        else:
            im = ts.images[int(rec["index"][b, 0])]
            want = im["hw"] + (im["image_id"],)
        assert (int(img_info[0][b]), int(img_info[1][b]), int(img_id[b, 0])) == want, b
    return imgs, targets


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["lmo", "tless"])
def test_whole_batch_matches_the_oracle(dev, which, request):
    root, cfg = request.getfixturevalue(which)
    bt = YT.YoloxTrainBatcher(cfg, root, seed=11, device=dev)
    try:
        assert bt.batch_size == 32
        _check_batch(bt, bt.ts, cfg.aug_wrapper["FORMAT"])
        assert bt.last_records["mosaic"].all() and bt.last_records["do_color"].any() and bt.last_records["mixup"].any()
        bt.close_mosaic()
        _check_batch(bt, bt.ts, cfg.aug_wrapper["FORMAT"])
        assert not bt.last_records["mosaic"].any()
    finally:
        bt.close()


@pytest.mark.gpu
def test_same_seed_same_batches(dev, lmo):
    root, cfg = lmo
    out = []
    for _ in range(2):
        bt = YT.YoloxTrainBatcher(cfg, root, seed=4, batch_size=8, device=dev)
        try:
            out.append([next(bt)[:2] for _ in range(2)])
        finally:
            bt.close()
    for (a_i, a_t), (b_i, b_t) in zip(*out):
        assert a_i.equal(b_i) and a_t.equal(b_t)
