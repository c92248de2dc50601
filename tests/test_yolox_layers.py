"""The YOLOX network one step of its layer plan at a time (yolox_model_run_step: the forward's own step function and
kernels) against float64 / float32 torch references of the same op, in both precision modes.

The engine describes its plan (yolox_model_plan_info / yolox_model_step_info): every step's kind, packed conv name, source /
destination / residual buffer with channel offset and count, map sizes, kernel size, stride and activation.  On the host,
that table replayed through oracle.yolox_oracle.replay_step in float64 reproduces the oracle forward; so the table, the
merged head convs and the interpreter the GPU tests rely on are checked without a GPU.

On the GPU every step of the forward runs in order.  Before each step the whole workspace is snapshotted; after it:
  * the destination slice is compared with the reference op applied to the kernel's own input, read from the snapshot
    (errors do not accumulate from step to step);
  * every other byte of the workspace, and every det_preds row outside the step's level, is unchanged;
  * the step, run again from the snapshot, gives bit-identical output (the shortcut add is in place, so the snapshot is
    restored first).
The walk's det_preds then equal yolox_model_forward's bit for bit (and a TTA plan's rows those of forward_tta).

Conv reference per mode (packed weights restated independently of the engine: oracle.yolox_oracle.packed_conv):
  * bf16x3: the fp64 conv of the fp32 input with the fp64 folded weights.
  * bf16:   the same with the input rounded to bf16 and the folded weights rounded fp64 -> fp32 -> bf16, as the engine
            packs them; the bias is the fp32 bias the kernel reads.
Error = max |got - ref| / max(1, max |ref|).  Focus, SPP, upsample and the head output are compared bit for bit with
torch fp32 on the same input (ULPS: the largest difference allowed, in units in the last place).

Configs: each covers shapes the others miss.
  x_256x320  depth 1.33 width 1.25, 8 classes, B=2: every YOLOX-X channel count (80 ... 1280, none a multiple of 64), K
             tails such as 9*80 = 720, the 12-bottleneck CSPs.
  s_480x640  0.33 / 0.5, 21 classes, B=1: the 15 x 20 level, partial 128-row tiles.
  t_64x96    0.33 / 0.375, 1 class, B=5: 24-channel layers (K = 24, less than one 32-wide k-chunk), 2 x 3 maps whose
             128-row tiles span all 5 images, a cls conv with N = 1.
  m_128x160  0.67 / 0.75, 30 classes, B=3: 48-channel layers.
Each state dict is calibrated at its own input size (make_yolox_state_dict, as test_yolox does).

Targeted inputs on selected conv steps, written into the source slice through the buffer view: "halo" (a per-image offset
and 3x the amplitude in the outermost rows and columns, so a tap read from a neighbouring image or across the zero padding
shows) and "large" (the input scaled so that the pre-activations reach +-100: SiLU's __expf / __fdividef tails).
"""
import ctypes

import pytest
import torch
from test_yolox import _f64, _synthetic

from gdrnpp_bop2022_b200 import _lib
from gdrnpp_bop2022_b200.yolox_model import YOLOX, _Engine
from oracle import yolox_oracle as O
from oracle import yolox_tta_oracle as T

MODES = ("bf16x3", "bf16")
CONFIGS = {   # name: depth, width, num_classes, (H, W), B (= max_batch)
    "x_256x320": (1.33, 1.25, 8, (256, 320), 2),
    "s_480x640": (0.33, 0.5, 21, (480, 640), 1),
    "t_64x96": (0.33, 0.375, 1, (64, 96), 5),
    "m_128x160": (0.67, 0.75, 30, (128, 160), 3),
}
TTA_SCALES = (1, 0.75, 1.25)   # plan 1: 48 x 72 content in 64 x 96 (downsampling); plan 2: 80 x 120 in 96 x 128 (upsampling)

# (quantity, mode) -> bar, with the largest error measured over all cases of the quantity (H100 80GB HBM3, 700 W power
# limit) and where it occurred.  "conv" covers every conv step of plan 0 of the four configs and of the two TTA plans.
BARS = {
    ("conv", "bf16x3"): 9e-5,    # 2.30e-5  x_256x320 backbone.bu_conv1
    ("conv", "bf16"): 2.8e-5,    # 7.19e-6  x_256x320 backbone.bu_conv1 (bf16 operands of the reference too: fp32 sums only)
    ("halo", "bf16x3"): 8e-5,    # 2.03e-5  x_256x320 backbone.C3_n4.m.0.conv2
    ("halo", "bf16"): 2.4e-5,    # 6.20e-6  x_256x320 backbone.C3_n4.m.0.conv2
    ("large", "bf16x3"): 9.5e-5,   # 2.42e-5  x_256x320 backbone.bu_conv1
    ("large", "bf16"): 3.3e-5,   # 8.26e-6  x_256x320 backbone.bu_conv1
}
# step kind -> largest difference from torch fp32 allowed, in units in the last place.  Every one measured 0: Focus and
# the upsample are copies, SPP a max, the head output and the TTA resample follow torch's fp32 operations one for one.
ULPS = {"focus": 0, "focus_resample": 0, "spp": 0, "upsample": 0, "head": 0}

TARGETED = ("backbone.backbone.stem.conv", "backbone.backbone.dark2.0", "backbone.backbone.dark3.1.m.0.conv2",
            "backbone.backbone.dark5.0", "backbone.backbone.dark5.1.conv2", "backbone.C3_n4.m.0.conv2", "backbone.bu_conv1",
            "head.conv0.0", "head.conv0.2", "head.cls_convs.2.1", "head.regobj.2", "head.cls.2")


# ------------------------------------------------------------------------------------------------------------- host
def _host_engine(depth, width, nc, H, W, max_batch=2):
    """A weightless engine: plans and step tables only (host only, no device call)."""
    return _Engine(YOLOX(depth, width, nc, max_batch=max_batch), "cpu", H, W, load=False)


def _replay(eng, plan, sd64, x, scale, det):
    """Replay a plan's step table in float64 on the host: buffers [B, pix, ld] of zeros, weights by packed name."""
    B = x.shape[0]
    info = eng.plan_info(plan)
    bufs = []
    for i in range(info["n_bufs"]):
        _, pix, ld, _ = eng.buffer_info(plan, i, B)
        bufs.append(torch.zeros(B, pix, ld, dtype=torch.float64))
    steps = eng.steps(plan)
    weights = {s["name"]: O.packed_conv(sd64, s["name"]) for s in steps if s["kind"] == "conv"}
    for s in steps:
        O.replay_step(s, bufs, x, det, weights, scale, info["a_base"])
    return steps


@pytest.mark.parametrize("fused", [False, True])
def test_step_table_replays_the_oracle_forward(lib, fused):
    from gdrnpp_bop2022_b200.synthetic import make_yolox_state_dict

    depth, width, nc, (H, W) = 0.33, 0.25, 3, (64, 96)
    sd = make_yolox_state_dict(O.yolox_forward, depth, width, nc, seed=0, calib_hw=(H, W), calib_batch=4)
    if fused:   # a fuse_model state dict: conv biases, no BatchNorm
        m = YOLOX(depth, width, nc)
        m.load_state_dict(sd)
        sd = m.fuse().state_dict()
    sd64 = _f64(sd)
    x = torch.rand((2, 3, H, W), generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 255
    eng = _host_engine(depth, width, nc, H, W)
    det = torch.zeros(2, eng.A, 5 + nc, dtype=torch.float64)
    steps = _replay(eng, 0, sd64, x, 1.0, det)
    ref = O.yolox_forward(sd64, x, depth, nc)
    assert (det - ref).abs().max().item() < 1e-10
    # the table: 1 Focus, 1 SPP, 2 upsamples, 3 head outputs, the rest convs; every slot within its buffer
    kinds = [s["kind"] for s in steps]
    assert (kinds.count("focus"), kinds.count("spp"), kinds.count("upsample"), kinds.count("head")) == (1, 1, 2, 3)
    assert kinds[0] == "focus" and kinds[-1] == "head"
    for s in steps:
        assert s["s_c"] > 0 and s["d_c"] > 0, s
        for buf, off, c in ((s["src"], s["s_off"], s["s_c"]), (s["dst"], s["d_off"], s["d_c"]), (s["res"], s["r_off"], s["d_c"])):
            if buf >= 0:
                assert off >= 0 and off + c <= eng.buffer_info(0, buf, 2)[2], s
    names = {s["name"] for s in steps if s["kind"] == "conv"}
    assert {"head.conv0.0", "head.regobj.1", "head.cls.2", "backbone.backbone.stem.conv"} <= names
    conv0 = next(s for s in steps if s["name"] == "head.conv0.0")
    assert (conv0["d_c"], conv0["ks"], conv0["act"]) == (128, 3, 1)
    for s in steps:
        if s["name"].startswith(("head.regobj.", "head.cls.")):
            assert s["act"] == 0 and s["ks"] == 1 and s["d_c"] == (5 if "regobj" in s["name"] else nc)

    # the test-time-augmentation plans: rows [a_base, a_base + A) of the TTA forward
    eng.set_scales(TTA_SCALES)
    ref = T.yolox_forward_tta(sd64, x, depth, nc, TTA_SCALES)
    for plan, s in ((1, 0.75), (2, 1.25)):
        info = eng.plan_info(plan)
        assert info["A_row"] == eng.A_tta == ref.shape[1]
        det = torch.zeros(2, info["A_row"], 5 + nc, dtype=torch.float64)
        _replay(eng, plan, sd64, x, s, det)
        rows = slice(info["a_base"], info["a_base"] + info["A"])
        assert (det[:, rows] - ref[:, rows]).abs().max().item() < 1e-10, plan


def test_step_table_entries_reject_bad_arguments(lib):
    eng = _host_engine(0.33, 0.25, 3, 64, 96, max_batch=2)
    h, info, name = eng.handle, (ctypes.c_int * 18)(), ctypes.create_string_buffer(256)
    n = eng.plan_info(0)["n_steps"]
    i64 = (ctypes.c_int64 * 4)()
    assert lib.yolox_model_plan_info(h, 1, info) != 0                    # no scale set: plan 0 only
    assert lib.yolox_model_plan_info(h, -1, info) != 0
    assert lib.yolox_model_step_info(h, 0, n, info, name, 256) != 0
    assert lib.yolox_model_step_info(h, 0, -1, info, name, 256) != 0
    assert lib.yolox_model_step_info(h, 0, 1, info, name, 4) != 0        # "backbone.backbone.stem.conv" does not fit
    assert lib.yolox_model_step_info(h, 0, 0, info, name, 1) == 0 and name.value == b""   # Focus has no name
    assert lib.yolox_model_buffer_info(h, 0, eng.plan_info(0)["n_bufs"], 1, i64) != 0
    assert lib.yolox_model_buffer_info(h, 0, 0, 3, i64) != 0              # batch above max_batch
    assert lib.yolox_model_buffer_info(h, 0, 0, 0, i64) != 0
    # run_step rejects before touching a pointer: these are never dereferenced
    p = ctypes.c_void_p(1 << 20)
    ws = eng.buffer_info(0, 0, 2)[3]
    assert lib.yolox_model_run_step(h, 0, 0, p, 2, p, p, ws, None) != 0   # no weights loaded
    assert b"weights missing" in lib.gdrn_last_error()
    for plan, step, batch in ((1, 0, 1), (0, n, 1), (0, -1, 1), (0, 0, 3), (0, 0, 0)):
        assert lib.yolox_model_run_step(h, plan, step, p, batch, p, p, ws, None) != 0, (plan, step, batch)
    assert lib.yolox_model_run_step(h, 0, 0, None, 1, p, p, ws, None) != 0
    eng.set_scales(TTA_SCALES)
    assert eng.plan_info(2)["a_base"] == eng.plan_info(0)["A"] + eng.plan_info(1)["A"]
    assert lib.yolox_model_plan_info(h, 3, info) != 0


# ------------------------------------------------------------------------------------------------------------- GPU
_CACHE = {}


def _setup(cfg, mode):
    depth, width, nc, hw, B = CONFIGS[cfg]
    if cfg not in _CACHE:
        sd = _synthetic(depth, width, nc, hw, 32 if hw[0] < 100 else 2)
        _CACHE.clear()   # one config's weights on the device at a time
        _CACHE[cfg] = (sd, _f64(sd, "cuda"), {})
    sd, sd64, weights = _CACHE[cfg]
    m = YOLOX(depth, width, nc, max_batch=B, precision=mode).eval()
    m.load_state_dict(sd)
    m.cuda()
    eng = m._engine(torch.device("cuda", 0), *hw)
    for s in eng.steps(0):
        if s["kind"] == "conv" and s["name"] not in weights:
            weights[s["name"]] = O.packed_conv(sd64, s["name"])
    return m, eng, weights


def _image(B, hw, seed):
    return (torch.rand((B, 3) + tuple(hw), generator=torch.Generator().manual_seed(seed)) * 255).cuda()


def _err(got, ref):
    got, ref = got.double(), ref.double()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _ulps(got, ref):
    """Largest difference in units in the last place between two fp32 tensors (0 when bit-identical)."""
    if torch.equal(got.contiguous().view(torch.int32), ref.contiguous().view(torch.int32)):
        return 0
    gi, ri = got.contiguous().view(torch.int32).long(), ref.contiguous().view(torch.int32).long()
    gi = torch.where(gi < 0, -(gi & 0x7FFFFFFF), gi)   # sign-magnitude -> ordered integers
    ri = torch.where(ri < 0, -(ri & 0x7FFFFFFF), ri)
    return int((gi - ri).abs().max().item())


def _conv_ref(s, views, w, b, mode):
    inp = O.nchw(views[s["src"]], s["s_off"], s["s_c"], s["in_h"], s["in_w"]).double()
    res = None
    if s["res"] >= 0:
        res = O.nchw(views[s["res"]], s["r_off"], s["d_c"], s["out_h"], s["out_w"]).double()
    if mode == "bf16":
        inp = inp.float().bfloat16().double()
        w, b = w.float().bfloat16().double(), b.float().double()
    return O.conv_op(inp, w, b, s["stride"], s["act"], res)


def _check_step(eng, plan, i, s, x, det, ws, views, weights, mode, scale, a_base):
    """Run step i once from the current workspace and check it (see the module docstring) -> (quantity, error or ulps)."""
    if s["kind"] == "head":
        a0 = a_base + s["anchor_off"]
        region = lambda: det[:, a0:a0 + s["in_h"] * s["in_w"]]  # noqa: E731
    else:
        region = lambda: O.nchw(views[s["dst"]], s["d_off"], s["d_c"], s["out_h"], s["out_w"])  # noqa: E731
    before, snap, det0 = region().clone(), ws.clone(), det.clone()
    eng.run_step(x, det, ws, plan, i)
    got = region().clone()
    region().copy_(before)   # back to the snapshot: nothing else may have changed
    assert torch.equal(ws, snap), ("workspace written outside the step's slice", plan, i, s)
    assert torch.equal(det, det0), ("det_preds written outside the step's rows", plan, i, s)
    k = s["kind"]
    if k == "conv":
        w, b = weights[s["name"]]
        q, e = "conv", _err(got, _conv_ref(s, views, w, b, mode))
    elif k == "focus":
        q = "focus" if scale == 1 else "focus_resample"
        e = _ulps(got, O.focus_op(T.tta_scale_input(x, scale).float()))
    elif k == "spp":
        e, q = _ulps(got, O.spp_op(O.nchw(views[s["src"]], 0, s["s_c"], s["in_h"], s["in_w"]))), "spp"
    elif k == "upsample":
        e, q = _ulps(got, O.upsample_op(O.nchw(views[s["src"]], s["s_off"], s["s_c"], s["in_h"], s["in_w"]))), "upsample"
    else:
        inv = float(torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(scale), dtype=torch.float32))
        raw = O.nchw(views[s["src"]], 0, s["s_c"], s["in_h"], s["in_w"])
        e, q = _ulps(got, O.head_op(raw, s["level_stride"], inv)), "head"
    eng.run_step(x, det, ws, plan, i)
    assert torch.equal(region(), got), ("a second run from the snapshot differs", plan, i, s)
    return q, e


def _walk(eng, plan, x, det, ws, weights, mode, scale, label):
    """Every step of a plan in order, each checked; -> {quantity: (max error, step name)}."""
    B = x.shape[0]
    info = eng.plan_info(plan)
    views = [eng.buffer(ws, plan, j, B) for j in range(info["n_bufs"])]
    worst = {}
    for i, s in enumerate(eng.steps(plan)):
        q, e = _check_step(eng, plan, i, s, x, det, ws, views, weights, mode, scale, info["a_base"])
        if q not in worst or e > worst[q][0]:
            worst[q] = (e, s["name"] or f"{s['kind']} {i}")
    for q, (e, where) in sorted(worst.items()):
        print(f"{label} plan {plan}: {q} max {e:.3g} at {where}")
    return worst


def _assert_worst(worst, mode):
    for q, (e, where) in worst.items():
        if q in ULPS:
            assert e <= ULPS[q], (q, e, where)
        else:
            assert e <= BARS[(q, mode)], (q, mode, e, where)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_every_step_of_the_forward(cfg, mode):
    depth, width, nc, hw, B = CONFIGS[cfg]
    m, eng, weights = _setup(cfg, mode)
    x = _image(B, hw, 5)
    det = torch.full((B, eng.A, 5 + nc), -7.0, device="cuda")
    ws = eng.new_workspace(B)
    worst = _walk(eng, 0, x, det, ws, weights, mode, 1.0, f"{cfg} {mode}")
    _assert_worst(worst, mode)
    # the chain of steps is the forward, bit for bit
    torch.cuda.synchronize()
    assert torch.equal(det, m(x)["det_preds"])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_tta_plans_step_by_step(mode):
    cfg = "t_64x96"
    depth, width, nc, hw, B = CONFIGS[cfg]
    m, eng, weights = _setup(cfg, mode)
    x = _image(B, hw, 6)
    ref = m(x, augment=True, cfg={"scales": TTA_SCALES})["det_preds"]
    det = torch.full_like(ref, -7.0)
    ws = eng.new_workspace(B, tta=True)
    for plan, scale in ((1, 0.75), (2, 1.25)):
        info = eng.plan_info(plan)
        assert (info["A_row"], info["H"], info["W"]) == (ref.shape[1],) + T.tta_sizes(*hw, scale)[1]
        worst = _walk(eng, plan, x, det, ws, weights, mode, scale, f"{cfg} {mode} scale {scale}")
        _assert_worst(worst, mode)
        rows = slice(info["a_base"], info["a_base"] + info["A"])
        assert torch.equal(det[:, rows], ref[:, rows]), plan


def _targeted_input(kind, s, w, B, g):
    c, h, wd = s["s_c"], s["in_h"], s["in_w"]
    v = torch.randn((B, c, h, wd), generator=g, dtype=torch.float64)
    if kind == "halo":
        v = v + torch.linspace(-3.0, 4.0, B, dtype=torch.float64)[:, None, None, None]
        v[:, :, [0, -1], :] *= 3.0
        v[:, :, :, [0, -1]] *= 3.0
    else:   # pre-activations (without the bias) up to +-100
        y = torch.nn.functional.conv2d(v.cuda(), w, stride=s["stride"], padding=(s["ks"] - 1) // 2)
        v = v * (100.0 / y.abs().max().item())
    return v.float().cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_targeted_conv_inputs(cfg, mode):
    depth, width, nc, hw, B = CONFIGS[cfg]
    m, eng, weights = _setup(cfg, mode)
    x = _image(B, hw, 7)
    det = torch.zeros((B, eng.A, 5 + nc), device="cuda")
    ws = eng.new_workspace(B)
    ws.zero_()
    views = [eng.buffer(ws, 0, j, B) for j in range(eng.plan_info(0)["n_bufs"])]
    g = torch.Generator().manual_seed(11)
    steps = [(i, s) for i, s in enumerate(eng.steps(0)) if s["name"] in TARGETED]
    assert len(steps) == len(TARGETED)
    worst = {}
    for i, s in steps:
        w, _ = weights[s["name"]]
        for kind in ("halo", "large"):
            O.store(views[s["src"]], s["s_off"], _targeted_input(kind, s, w, B, g))
            if s["res"] >= 0:
                O.store(views[s["res"]], s["r_off"], torch.randn((B, s["d_c"], s["out_h"], s["out_w"]), generator=g).cuda())
            _, e = _check_step(eng, 0, i, s, x, det, ws, views, weights, mode, 1.0, 0)
            if kind not in worst or e > worst[kind][0]:
                worst[kind] = (e, s["name"])
    for q, (e, where) in sorted(worst.items()):
        print(f"{cfg} {mode} targeted: {q} max {e:.3g} at {where}")
    _assert_worst(worst, mode)


@pytest.mark.gpu
def test_run_step_rejects_bad_arguments():
    cfg = "t_64x96"
    m, eng, _ = _setup(cfg, "bf16x3")
    depth, width, nc, hw, B = CONFIGS[cfg]
    L = _lib.lib()
    x = _image(B, hw, 8)
    det = torch.zeros((B, eng.A, 5 + nc), device="cuda")
    ws = eng.new_workspace(B)
    need = eng.buffer_info(0, 0, B)[3]
    assert ws.numel() >= need
    st = _lib.current_stream()
    run = lambda plan, step, b, nbytes: L.yolox_model_run_step(eng.handle, plan, step, _lib.ptr(x), b, _lib.ptr(det),  # noqa: E731
                                                               _lib.ptr(ws), nbytes, st)
    n = eng.plan_info(0)["n_steps"]
    assert run(0, 0, B, need) == 0
    assert run(0, 0, B, need - 1) != 0 and b"workspace too small" in L.gdrn_last_error()
    assert run(0, n, B, need) != 0 and run(0, -1, B, need) != 0
    assert run(1, 0, B, need) != 0                       # no scale set yet
    assert run(0, 0, B + 1, need) != 0 and run(0, 0, 0, need) != 0
    with pytest.raises(_lib.GdrnError):
        eng.buffer(ws[:need - 1], 0, 0, B)
    torch.cuda.synchronize()
