"""YOLOX multi-scale test-time augmentation (YOLOX.forward(augment=True, cfg), test.augment / test.scales of the shipped
BOP test configs): the oracle against the reference fixture, the scaled sizes, the config reader and the argument checks
on the host; the CUDA forward against the fp64 oracle, its exact relations to the plain forward, graph replay and the
predictor on the GPU."""
import ctypes
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_ref_yolox import draw_state_dict  # noqa: E402
from test_yolox import BARS, BASE_CFG, DERIVED_CFG, _errs, _f64, _scene, _synthetic  # noqa: E402

from gdrnpp_bop2022_b200 import _lib  # noqa: E402
from gdrnpp_bop2022_b200.yolox_model import YOLOX, load_yolox_config  # noqa: E402
from oracle import yolox_oracle as O  # noqa: E402
from oracle import yolox_tta_oracle as T  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "ref_yolox_tta.npz")
SHIPPED = (1, 0.75, 0.83, 1.12, 1.25)   # test.scales of every configs/yolox/bop_pbr/yolox_x_640_* config


def _gold():
    z = np.load(GOLD)
    return z, draw_state_dict(list(z["names"]), list(z["shapes"]))


def _anchors(ph, pw):
    return sum((ph // s) * (pw // s) for s in (8, 16, 32))


def test_oracle_tta_reproduces_reference_fixture():
    z, sd = _gold()
    assert tuple(z["scales"]) == SHIPPED
    out = T.yolox_forward_tta(_f64(sd), torch.from_numpy(z["x"]).double(), float(z["depth"]), int(z["num_classes"]), SHIPPED)
    ref = torch.from_numpy(z["det_preds"]).double()
    assert out.shape == ref.shape == (2, 882, 8)
    # the fixture is the reference's fp32 forward: agreement to fp32 round-off
    assert torch.allclose(out, ref, rtol=1e-5, atol=2e-5), (out - ref).abs().max()


@pytest.mark.parametrize("h,w", [(640, 640), (480, 640), (64, 96), (96, 64), (352, 608), (1024, 1280)])
def test_scaled_sizes_and_anchor_count(lib, h, w):
    scales = (1, 0.75, 0.83, 1.12, 1.25, 0.5, 0.6, 0.7, 0.9, 1.1, 1.3, 1.33, 1.5, 2.0)
    expect_a = 0
    for s in scales:
        (ch, cw), (ph, pw) = T.tta_sizes(h, w, s)
        # the scaled input the oracle builds: content int(h*s) x int(w*s) (the only unpadded rows / columns), padded to
        # ceil(h*s/32)*32 x ceil(w*s/32)*32
        xi = T.tta_scale_input(torch.zeros(1, 3, h, w), s)
        assert xi.shape[-2:] == (ph, pw) and ph % 32 == 0 and pw % 32 == 0
        if s != 1:
            assert (ch, cw) == (int(h * s), int(w * s))
            assert int((xi[0, 0, :, 0] == 0).sum()) == ch and int((xi[0, 0, 0, :] == 0).sum()) == cw
        expect_a += _anchors(ph, pw)
    # the engine lays its plans out from the same sizes (host only, no device call)
    h_ = ctypes.c_void_p()
    _lib.check(lib.yolox_model_create(ctypes.byref(h_), 0.33, 0.25, 3, 2, h, w, 1), "yolox_model_create")
    try:
        _lib.check(lib.yolox_model_set_scales(h_, (ctypes.c_double * len(scales))(*scales), len(scales)), "set_scales")
        assert lib.yolox_model_num_anchors_tta(h_) == expect_a
        assert lib.yolox_model_num_anchors(h_) == _anchors(h, w)   # plan 0 is untouched
        one = (ctypes.c_double * 1)(1.0)
        _lib.check(lib.yolox_model_set_scales(h_, one, 1), "set_scales")   # a new set replaces the old one
        assert lib.yolox_model_num_anchors_tta(h_) == _anchors(h, w)
        bad = (ctypes.c_double * 2)(1.0, 0.5 / min(h, w))   # int(h*s) or int(w*s) is 0
        assert lib.yolox_model_set_scales(h_, bad, 2) != 0
        assert lib.yolox_model_num_anchors_tta(h_) == _anchors(h, w)   # a rejected set leaves the current one
    finally:
        lib.yolox_model_destroy(h_)


def test_shipped_sizes_at_640():
    sizes = [T.tta_sizes(640, 640, s) for s in SHIPPED]
    assert [p[0] for _, p in sizes] == [640, 480, 544, 736, 800]
    assert [c[0] for c, _ in sizes] == [640, 480, 531, 716, 800]
    assert sum(_anchors(*p) for _, p in sizes) == 43428
    # at the fixture's 64 x 96: two network sizes, contents 48 x 72, 53 x 79, 71 x 107, 80 x 120
    sizes = [T.tta_sizes(64, 96, s) for s in SHIPPED]
    assert [c for c, _ in sizes[1:]] == [(48, 72), (53, 79), (71, 107), (80, 120)]
    assert [p for _, p in sizes] == [(64, 96)] * 3 + [(96, 128)] * 2
    assert sum(_anchors(*p) for _, p in sizes) == 882


def test_load_yolox_config_tta_fields(tmp_path):
    (tmp_path / "yolox_base.py").write_text(BASE_CFG)
    (tmp_path / "yolox_x_lmo.py").write_text(DERIVED_CFG)
    c = load_yolox_config(str(tmp_path / "yolox_x_lmo.py"))
    assert (c.augment, c.scales) == (True, SHIPPED)
    assert (c.depth, c.width, c.num_classes, c.test_size, c.conf_thr, c.nms_thr) == (1.33, 1.25, 8, (640, 640), 0.001, 0.65)
    c = load_yolox_config(str(tmp_path / "yolox_base.py"))
    assert (c.augment, c.scales) == (False, None)
    # the keys inside the test = dict(...) of a base config are read too
    (tmp_path / "yolox_base.py").write_text(BASE_CFG.replace("half_test=True,", "half_test=True, augment=True, scales=(1, 0.5),"))
    c = load_yolox_config(str(tmp_path / "yolox_base.py"))
    assert (c.augment, c.scales) == (True, (1, 0.5))


@pytest.mark.skipif(not os.environ.get("GDRN_REFERENCE_SRC"), reason="GDRN_REFERENCE_SRC not set")
def test_shipped_configs_ask_for_tta():
    import glob

    files = sorted(glob.glob(os.path.join(os.environ["GDRN_REFERENCE_SRC"], "configs", "yolox", "bop_pbr", "yolox_x_*.py")))
    assert files
    for f in files:
        c = load_yolox_config(f)
        assert (c.augment, c.scales) == (True, SHIPPED), f


def test_augment_needs_scales():
    m = YOLOX(0.33, 0.25, 3).eval()
    x = torch.zeros(1, 3, 64, 96)
    for cfg in (None, SimpleNamespace(), SimpleNamespace(scales=None), {}, {"scales": None}):
        with pytest.raises(NotImplementedError):
            m(x, augment=True, cfg=cfg)


# ------------------------------------------------------------------------------------------------------------- GPU
def _model(depth, width, nc, sd, precision="bf16x3", max_batch=8):
    m = YOLOX(depth, width, nc, max_batch=max_batch, precision=precision).eval()
    m.load_state_dict(sd)
    return m.cuda()


def _tta(m, x, scales=SHIPPED):
    return m(x, augment=True, cfg=SimpleNamespace(scales=scales))["det_preds"]


@pytest.mark.gpu
def test_reference_fixture_tta_on_gpu():
    z, sd = _gold()
    depth, width, nc = float(z["depth"]), float(z["width"]), int(z["num_classes"])
    ref = T.yolox_forward_tta(_f64(sd), torch.from_numpy(z["x"]).double(), depth, nc, SHIPPED)
    for precision, (box_tol, score_tol) in BARS.items():
        out = _tta(_model(depth, width, nc, sd, precision), torch.from_numpy(z["x"]).cuda())
        assert out.shape == ref.shape
        eb, es = _errs(out, ref)
        print(f"reference fixture TTA {precision}: box {eb:.3g} px score {es:.3g}")
        assert eb < box_tol and es < score_tol, (precision, eb, es)
        # and the reference's own fp32 output, within the same bars
        eb, es = _errs(out, torch.from_numpy(z["det_preds"]).double())
        assert eb < box_tol and es < score_tol, ("fixture", precision, eb, es)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2])
def test_yolox_x_640_tta_against_fp64_oracle(B):
    sd = _synthetic(1.33, 1.25, 8, (640, 640), 2)
    x = torch.rand((B, 3, 640, 640), generator=torch.Generator().manual_seed(17)) * 255
    ref = T.yolox_forward_tta(_f64(sd, "cuda"), x.double().cuda(), 1.33, 8, SHIPPED)
    for precision, (box_tol, score_tol) in BARS.items():
        m = _model(1.33, 1.25, 8, sd, precision)
        out = _tta(m, x.cuda())
        assert out.shape == (B, 43428, 13)
        assert m._engines[(640, 640)].A_tta == 43428
        eb, es = _errs(out, ref)
        print(f"YOLOX-X 640x640 TTA B={B} {precision}: max box err {eb:.3g} px, max score err {es:.3g}")
        assert eb < box_tol and es < score_tol, (precision, eb, es)
        del m


@pytest.mark.gpu
def test_small_tta_in_chunks():
    sd = _synthetic(0.33, 0.25, 8, (480, 640), 2)
    x = torch.rand((5, 3, 480, 640), generator=torch.Generator().manual_seed(18)) * 255
    ref = T.yolox_forward_tta(_f64(sd, "cuda"), x.double().cuda(), 0.33, 8, SHIPPED)
    for precision, (box_tol, score_tol) in BARS.items():
        out = _tta(_model(0.33, 0.25, 8, sd, precision, max_batch=2), x.cuda())   # B = 5 in chunks of 2
        eb, es = _errs(out, ref)
        print(f"width 0.25 480x640 B=5 TTA {precision}: box {eb:.3g} px score {es:.3g}")
        assert eb < box_tol and es < score_tol, (precision, eb, es)


@pytest.mark.gpu
def test_tta_exact_relations_to_plain_forward():
    sd = _synthetic(0.33, 0.25, 8, (480, 640), 2)
    x = (torch.rand((3, 3, 480, 640), generator=torch.Generator().manual_seed(19)) * 255).cuda()
    for precision in BARS:
        m = _model(0.33, 0.25, 8, sd, precision, max_batch=2)
        plain = m(x)["det_preds"]
        A = plain.shape[1]
        out = _tta(m, x)
        assert torch.equal(out[:, :A], plain)                      # the scale-1 slice is the plain forward
        assert torch.equal(_tta(m, x, (1,)), plain)                # scales = (1,) is the plain forward
        a075 = _anchors(*T.tta_sizes(480, 640, 0.75)[1])
        assert torch.equal(_tta(m, x, (0.75, 1)), torch.cat([out[:, A:A + a075], plain], 1))   # any order, same rows
        again = m(x)["det_preds"]                                  # plain after TTA: a fresh model's output
        fresh = _model(0.33, 0.25, 8, sd, precision, max_batch=2)(x)["det_preds"]
        assert torch.equal(again, fresh) and torch.equal(again, plain)
        assert len(m._engines) == 1                                # one engine, one weight copy, for every size
        del m


@pytest.mark.gpu
def test_tta_determinism_batch_independence_and_graph():
    sd = _synthetic(0.33, 0.25, 8, (480, 640), 2)
    x = (torch.rand((5, 3, 480, 640), generator=torch.Generator().manual_seed(20)) * 255).cuda()
    m = _model(0.33, 0.25, 8, sd, max_batch=5)
    a = _tta(m, x)
    assert torch.equal(a, _tta(m, x))
    for i in (0, 3):
        assert torch.equal(_tta(m, x[i:i + 1].contiguous())[0], a[i])
    xs = x[:1].clone()
    replay, out = m.capture_graph(xs, augment=True, cfg={"scales": SHIPPED})
    xs.copy_(x[3:4])
    replay()
    torch.cuda.synchronize()
    assert torch.equal(out["det_preds"][0], a[3])
    # a plain forward and another scale set afterwards leave the graph's output as it was
    m(x)
    _tta(m, x, (1.25, 0.5))
    xs.copy_(x[4:5])
    replay()
    torch.cuda.synchronize()
    assert torch.equal(out["det_preds"][0], a[4])


@pytest.mark.gpu
def test_tta_errors():
    m = _model(0.33, 0.25, 3, _synthetic(0.33, 0.25, 3, (64, 96), 32))
    x = torch.zeros(1, 3, 64, 96, device="cuda")
    with pytest.raises(_lib.GdrnError):
        _tta(m, x, (1, 0.01))   # int(64 * 0.01) = 0: an empty scaled image
    m(x)
    eng = m._engines[(64, 96)]
    L = _lib.lib()
    det = torch.empty(1, eng.A, 8, device="cuda")
    ws = eng.new_workspace(1)
    # a fresh engine has no scale set: the TTA forward refuses to run
    h = ctypes.c_void_p()
    _lib.check(L.yolox_model_create(ctypes.byref(h), 0.33, 0.25, 3, 1, 64, 96, 1), "yolox_model_create")
    try:
        assert L.yolox_model_forward_tta(h, _lib.ptr(x), 1, _lib.ptr(det), _lib.ptr(ws), ws.numel(), _lib.current_stream()) != 0
        assert L.yolox_model_workspace_bytes_tta(h, 1) == 0 and L.yolox_model_num_anchors_tta(h) == 0
    finally:
        L.yolox_model_destroy(h)
    with pytest.raises(ValueError):
        _tta(m, x, ())


@pytest.mark.gpu
def test_predictor_tta_matches_oracle_pipeline():
    from gdrnpp_bop2022_b200.predictor_yolo import YoloPredictor, preproc

    sd = _synthetic(0.33, 0.5, 8, (640, 640), 2)
    cfg = SimpleNamespace(depth=0.33, width=0.5, num_classes=8, test_size=(640, 640), conf_thr=0.5, nms_thr=0.45,
                          augment=True, scales=SHIPPED)
    img = _scene(3, 480, 640)
    x, r = preproc(img, cfg.test_size)
    d = T.yolox_forward_tta(_f64(sd, "cuda"), torch.from_numpy(x)[None].double().cuda(), 0.33, 8, SHIPPED)[0].cpu().numpy()
    score = np.sort(d[:, 4] * d[:, 5:].max(1))
    # a threshold near 0.5 in a gap of the oracle scores, so that the comparison is well-posed
    gaps = [(abs(0.5 * (a + b) - 0.5), 0.5 * (a + b)) for a, b in zip(score[:-1], score[1:]) if b - a > 2e-3]
    cfg.conf_thr = float(min(gaps)[1])
    assert np.abs(score - cfg.conf_thr).min() > 1e-3, "an oracle score sits on the threshold"
    ious = []
    ref = O.keep_single_instance(d, 8, cfg.conf_thr, cfg.nms_thr, ious=ious)
    assert all(abs(v - cfg.nms_thr) > 1e-3 for v in ious), "a compared IoU sits on the NMS threshold"
    assert ref is not None
    for use_graph in (True, False):
        pred = YoloPredictor(cfg=cfg, state_dict=sd, augment=True, use_cuda_graph=use_graph)
        out = pred.inference(img)
        assert out[0] is not None
        got = out[0].cpu().numpy()
        assert got.shape == ref.shape, (got, ref)
        assert (got[:, 6] == ref[:, 6]).all()
        eb, es = np.abs(got[:, :4] - ref[:, :4] / r).max(), np.abs(got[:, 4:6] - ref[:, 4:6]).max()
        print(f"TTA predictor (graph {use_graph}) vs oracle pipeline: box err {eb:.3g}, score err {es:.3g}")
        assert eb < 0.05 and es < 1e-4
