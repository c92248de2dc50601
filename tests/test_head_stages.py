"""The geometry head and Patch-PnP one stage at a time (gdrn_model_run_stage: the forward's own stage functions, plans and
kernels) against float64 torch references of the same op, in both precision modes.

Reference per mode:
  * bf16x3: the fp64 op on the fp32 input and the fp32 weights -- the error includes the hi + lo representation.
  * bf16:   the fp64 op on the bf16-rounded input and bf16-rounded GEMM weights -- the error is accumulation order, the
            bf16 rounding of the stored outputs and (GroupNorm + GELU) the half2 tanh GELU.

Errors are in the scaled form of the GEMM tests, max |got - ref| / max(1, max |ref|).  Each bar is at most 4x the largest
error measured on an H100 (80GB HBM3, 400 W power limit) over all cases of the quantity; the measured maxima are listed
next to the bars in BARS.  The conv outputs before GroupNorm ("raw") of the split mode stay within the gdrn_gemm_x3 bar of
4e-5 (K <= 4096 here).

Inputs: every image carries its own offset (a read from a neighbouring image shows), the mean is non-zero and the
outermost rows and columns carry 3x the energy (wrong zero padding / TMA out-of-bounds fill shows).  Odd batches leave the
second image of the last 128-pixel box of the 8x8 maps beyond the batch; B = 5 is the per-image case with narrowed tiles,
B = 64 the bench batch.  Weights are seeded from a state dict owned by this file.
"""
import functools

import pytest
import torch
import torch.nn.functional as F

from oracle import gdrn_model_oracle as O

pytestmark = pytest.mark.gpu

MODES = ("bf16x3", "bf16")
BATCHES = (1, 3, 5, 64)
HEAD_STAGES = ("deconv",) + tuple(f"head_conv{i}" for i in range(6))
C3 = 1024                        # convnext_base backbone width
HEAD_IN_RES = {"deconv": 8, "head_conv0": 16, "head_conv1": 16, "head_conv2": 32, "head_conv3": 32, "head_conv4": 64,
               "head_conv5": 64}
GN_LAYER = {s: i for i, s in enumerate(HEAD_STAGES)}
GN_LAYER.update({f"pnp_conv{i}": 7 + i for i in range(3)})

# (quantity, mode) -> bar, with the largest error measured over all cases of the quantity (H100 80GB HBM3, 400 W power
# limit) and where it occurred.
BARS = {
    ("raw", "bf16x3"): 4e-5,      # 2.06e-5  deconv B=5 (K = 4 taps x 1024)
    ("raw", "bf16"): 1.2e-2,      # 3.16e-3  deconv B=5 (bf16 output rounding, 2^-9)
    ("gn_out", "bf16x3"): 4e-5,   # 1.22e-5  deconv B=64; 2.04e-5 in the |mean| / std = 100 case
    ("gn_out", "bf16"): 2.5e-2,   # 7.03e-3  head_conv3 B=64 (bf16 raw + half2 tanh GELU + bf16 upsample)
    ("gn_sums", "bf16x3"): 4e-7,  # 9.44e-8  pnp_conv2 B=64 sum of squares (fp32 per-warp partials), relative to sum |x|, sum x^2
    ("gn_sums", "bf16"): 4e-7,    # 1.08e-7  pnp_conv2 B=64 sum of squares
    ("pnp_in", "bf16x3"): 3e-5,   # 8.08e-6  B=5, class-aware
    ("pnp_in", "bf16"): 1.2e-2,   # 3.49e-3  B=3, class-aware (bf16 output rounding)
    ("maps", "bf16x3"): 2.5e-5,   # 6.84e-6  coor_z B=64
    ("maps", "bf16"): 1.6e-6,     # 4.36e-7  region B=5 (fp32 maps of the bf16 GEMM vs its bf16-rounded operands)
    ("fc", "bf16x3"): 2.4e-6,     # 6.10e-7  t_ B=17 (fp32 fc_f32 stack)
    ("fc", "bf16"): 2.5e-2,       # 6.73e-3  t_ B=17 (bf16 fc1 / fc2 activations)
}


def _err(got, ref):
    got, ref = got.double(), ref.double()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _assert_bars(errs, mode):
    for (what, q), e in errs.items():
        assert e <= BARS[(q, mode)], (what, q, mode, e, BARS[(q, mode)])


# ------------------------------------------------------------------------------------------------ fixtures
def _state_dict(num_classes, seed=0):
    """Seeded head / Patch-PnP weights at the scale of a trained network (He-initialised convs, GroupNorm affines near
    (1, 0)); the backbone is zero (no stage reads it)."""
    from gdrnpp_bop2022_b200.synthetic import state_dict_shapes

    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, s in state_dict_shapes("convnext_base", num_classes).items():
        if k.startswith("backbone."):
            sd[k] = torch.zeros(s)
        elif len(s) == 4:   # conv; ConvTranspose2d [Cin, Cout, 3, 3] sees Cin * 9 / 4 inputs per output on average
            fan = s[0] * 9 / 4 if k == "geo_head_net.features.0.weight" else s[1] * s[2] * s[3]
            sd[k] = torch.randn(s, generator=g) * (2.0 / fan) ** 0.5
        elif len(s) == 2:
            sd[k] = torch.randn(s, generator=g) * (2.0 / s[1]) ** 0.5
        elif k.endswith("weight"):   # GroupNorm gamma
            sd[k] = 1.0 + 0.2 * torch.randn(s, generator=g)
        else:
            sd[k] = 0.1 * torch.randn(s, generator=g)
    return sd


def _gn_ratio_weights(sd, li):
    """Head conv li with only the centre tap, W[o, i] = (1 + r[o, i] - mean_i r[o, i]) / 256: every output channel sums its
    256 inputs with total weight 1, so an input of mean c and unit spread gives groups of mean c and std ~ 0.088
    regardless of padding -- |mean| / std is set by c alone."""
    g = torch.Generator().manual_seed(100 + li)
    r = torch.randn(256, 256, generator=g)
    w = torch.zeros(256, 256, 3, 3)
    w[:, :, 1, 1] = (1.0 + r - r.mean(dim=1, keepdim=True)) / 256
    sd = dict(sd)
    sd[f"geo_head_net.features.{O.HEAD_CONVS[li]}.conv.weight"] = w
    return sd


@functools.lru_cache(maxsize=None)
def _setup(mode, num_classes=21, gn_ratio_conv=None):
    """(model, fp64 reference state dict) of one precision mode; class-agnostic for num_classes == 1."""
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg

    cfg = default_cfg(num_classes=21)
    if num_classes == 1:
        gh = cfg.MODEL.POSE_NET.GEO_HEAD
        gh.XYZ_CLASS_AWARE = gh.MASK_CLASS_AWARE = gh.REGION_CLASS_AWARE = False
    sd = _state_dict(num_classes)
    if gn_ratio_conv is not None:
        sd = _gn_ratio_weights(sd, gn_ratio_conv)
    model = GDRN_DoubleMask(cfg, max_batch=64, precision=mode)
    assert model.head_classes == num_classes
    model.load_state_dict(sd)
    dev = torch.device("cuda:0")
    ref_sd = {}
    for k, v in sd.items():
        if k.startswith("backbone."):
            continue
        if mode == "bf16" and v.dim() >= 2:   # GEMM operands are bf16 in this mode; vectors (bias, GN affine) stay fp32
            v = v.bfloat16().float()
        ref_sd[k] = v.double().to(dev)
    return model, ref_sd


def _input(shape, seed, edge_gain=3.0):
    """NHWC [B,H,W,C]: unit noise, 3x at the outermost rows / columns, mean 0.3 plus a per-image offset."""
    B, H, W, C = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    gain = torch.ones(H, W)
    gain[0, :] = gain[-1, :] = gain[:, 0] = gain[:, -1] = edge_gain
    off = 0.3 + 0.2 * ((torch.arange(B) * 5) % 7 - 3).float()
    return x * gain[None, :, :, None] + off[:, None, None, None]


def _ref_input(x, mode):
    x = x.bfloat16().float() if mode == "bf16" else x
    return x.double().cuda().permute(0, 3, 1, 2)   # NCHW


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _run_twice(model, stage, x, **kw):
    """Runs a stage twice on the same input: the outputs must be bit-identical.  (The GroupNorm sums are double atomics:
    their order may differ in the last bits of the double, below the float rounding of mean / rstd.)"""
    a = model.run_stage(stage, x, **kw)
    b = model.run_stage(stage, x, **kw)
    torch.cuda.synchronize()
    for k in a:
        if k == "gn_stats":
            assert (a[k] - b[k]).abs().max().item() <= 1e-12 * max(1.0, a[k].abs().max().item()), stage
        else:
            assert torch.equal(a[k], b[k]), (stage, k)
    return a


def _gn_sum_errors(stats, raw, layer, B):
    """The double GroupNorm sums [10,B,32,2] against fp64 sums of the conv output as stored; every other layer's slot
    (where a write for an image beyond the batch would land) stays zero."""
    x = raw.double().reshape(B, -1, 32, raw.shape[-1] // 32)
    s, ss = x.sum(dim=(1, 3)), (x * x).sum(dim=(1, 3))
    scale_s, scale_ss = x.abs().sum(dim=(1, 3)).clamp_min(1.0), ss.clamp_min(1.0)
    others = torch.cat([stats[:layer], stats[layer + 1:]])
    assert others.abs().max().item() == 0.0
    return {"sum": ((stats[layer, :, :, 0] - s).abs() / scale_s).max().item(),
            "sumsq": ((stats[layer, :, :, 1] - ss).abs() / scale_ss).max().item()}


# ------------------------------------------------------------------------------------------------ conv stages
def head_stage_errors(stage, mode, B, x=None):
    model, sd = _setup(mode)
    h = HEAD_IN_RES[stage]
    if x is None:
        x = _input((B, h, h, C3 if stage == "deconv" else 256), seed=10 * HEAD_STAGES.index(stage) + B)
    res = _run_twice(model, stage, x.cuda(), want_raw=True)
    xr = _ref_input(x, mode)
    with torch.no_grad():
        if stage == "deconv":
            ref, ref_raw = O.head_deconv(sd, xr)
        else:
            ref, ref_raw = O.head_conv(sd, xr, int(stage[-1]))
    errs = {(stage, "raw"): _err(_nchw(res["raw"]), ref_raw), (stage, "gn_out"): _err(_nchw(res["out"]), ref)}
    for k, e in _gn_sum_errors(res["gn_stats"], res["raw"], GN_LAYER[stage], B).items():
        errs[(stage + "." + k, "gn_sums")] = e
    return errs


def pnp_conv_errors(i, mode, B):
    model, sd = _setup(mode)
    stage = f"pnp_conv{i}"
    r = 64 >> i
    x = _input((B, r, r, 128), seed=50 + 7 * i + B)
    if i == 0:
        x[..., 69:] = 0.0   # the Patch-PnP input has 69 channels; the out conv writes zero pad columns
    res = _run_twice(model, stage, x.cuda(), want_raw=True)
    with torch.no_grad():
        ref, ref_raw = O.pnp_conv(sd, _ref_input(x, mode)[:, :69] if i == 0 else _ref_input(x, mode), i)
    errs = {(stage, "raw"): _err(_nchw(res["raw"]), ref_raw), (stage, "gn_out"): _err(_nchw(res["out"]), ref)}
    for k, e in _gn_sum_errors(res["gn_stats"], res["raw"], GN_LAYER[stage], B).items():
        errs[(stage + "." + k, "gn_sums")] = e
    return errs


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stage", HEAD_STAGES)
def test_head_stage_vs_fp64(dev, stage, mode, B):
    """Deconv (four parity GEMMs on rank-4 boxes, GNSTATS) and the six 3x3 head convs (nine-tap rank-4 plans; bilinear x2
    after convs 1 and 3): conv output, GroupNorm sums and GroupNorm + GELU (+ upsample) output."""
    _assert_bars(head_stage_errors(stage, mode, B), mode)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("i", [0, 1, 2])
def test_pnp_conv_vs_fp64(dev, i, mode, B):
    """Patch-PnP 3x3 s2 convs (rank-5 stride-2 view, parity taps, GNSTATS with 4 channels per group) + GroupNorm + GELU
    (gn_gelu_f32 for the last one in split mode)."""
    _assert_bars(pnp_conv_errors(i, mode, B), mode)


# ------------------------------------------------------------------------------------------------ out conv
LABELS = [-1, 21, 1000] + list(range(21))   # out of range values are clamped into [0, num_classes)


def out_conv_errors(mode, B, num_classes):
    model, sd = _setup(mode, num_classes)
    g = torch.Generator().manual_seed(300 + B + num_classes)
    x = _input((B, 64, 64, 256), seed=200 + B)
    ext = 0.05 + 0.3 * torch.rand(B, 3, generator=g)              # differs per axis and per ROI
    c2d = torch.rand(B, 2, 64, 64, generator=g) * 2 - 1
    labels = torch.tensor([LABELS[(7 * b + 3) % len(LABELS)] for b in range(B)], dtype=torch.int64)
    cls = labels if num_classes > 1 else None
    res = _run_twice(model, "out_conv", x.cuda(), roi_classes=None if cls is None else cls.cuda(), roi_extents=ext.cuda(),
                     roi_coord_2d=c2d.cuda(), want_maps=True)
    dev = torch.device("cuda:0")
    with torch.no_grad():
        out = F.conv2d(_ref_input(x, mode), sd["geo_head_net.out_layer.weight"], sd["geo_head_net.out_layer.bias"])
        nc = num_classes
        views = (out[:, :nc], out[:, nc:2 * nc], out[:, 2 * nc:3 * nc], out[:, 3 * nc:4 * nc], out[:, 4 * nc:5 * nc],
                 out[:, 5 * nc:])
        vis, full, cx, cy, cz, region = O.class_gather(*views, labels.clamp(0, nc - 1), num_classes=nc)
        coor = torch.cat([cx, cy, cz, c2d.double().to(dev)], dim=1)
        ref = O.pnp_input(coor, F.softmax(region[:, 1:], dim=1), ext.double().to(dev))
    pnp = res["out"]
    assert pnp[..., 69:].abs().max().item() == 0.0      # pad columns (and their lo halves) are exactly zero
    errs = {("pnp_in", "pnp_in"): _err(_nchw(pnp[..., :69]), ref)}
    for k, r in (("mask", vis), ("full_mask", full), ("coor_x", cx), ("coor_y", cy), ("coor_z", cz), ("region", region)):
        errs[(k, "maps")] = _err(res[k], r)
    return errs


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("num_classes", [21, 1])
def test_out_conv_vs_fp64(dev, num_classes, mode, B):
    """EPI_OUTCONV: class gather (labels covering all 21 classes plus out-of-range ones; class-agnostic head with NULL
    labels), NCHW maps, region softmax, (coord - 0.5) * extent, coord_2d, zero pad columns of the Patch-PnP input."""
    _assert_bars(out_conv_errors(mode, B, num_classes), mode)


# ------------------------------------------------------------------------------------------------ FC stack
def pnp_fc_errors(mode, B):
    model, sd = _setup(mode)
    g = torch.Generator().manual_seed(400 + B)
    x = torch.randn(B, 8, 8, 128, generator=g) * 0.6 + 0.1 * torch.arange(B)[:, None, None, None] % 0.7
    res = _run_twice(model, "pnp_fc", x.cuda())
    with torch.no_grad():
        rot, t = O.pnp_fc(sd, _ref_input(x, mode))    # the test permutes NHWC -> NCHW: pins pfc1's repacked columns
    out = res["out"]
    assert out[:, 9:].abs().max().item() == 0.0
    return {("rot6d", "fc"): _err(out[:, :6], rot), ("t_", "fc"): _err(out[:, 6:9], t)}


@pytest.mark.parametrize("B", [1, 16, 17, 20, 64])
@pytest.mark.parametrize("mode", MODES)
def test_pnp_fc_vs_fp64(dev, mode, B):
    """FC stack 8192 -> 1024 -> 256 -> 9 (fp32 split-K fc_f32 in split mode: B crosses its 16 / 64-row tiles and changes the
    K-slice count; GEMMs with GELU epilogues in bf16 mode); the 7 pad outputs stay exactly zero."""
    _assert_bars(pnp_fc_errors(mode, B), mode)


# ------------------------------------------------------------------------------------------------ GroupNorm, large mean
def gn_ratio_errors(mode, ratio, li=4, B=3):
    """Head conv li on groups with |mean| / std ~ ratio (see _gn_ratio_weights); returns the measured ratio and errors."""
    model, sd = _setup(mode, gn_ratio_conv=li)
    h = HEAD_IN_RES[f"head_conv{li}"]
    g = torch.Generator().manual_seed(500 + int(ratio))
    x = torch.randn(B, h, h, 256, generator=g) + ratio * 0.088
    errs = head_stage_errors(f"head_conv{li}", mode, B, x=x)
    with torch.no_grad():
        raw = O.head_conv(sd, _ref_input(x, mode), li)[1].reshape(B, 32, -1)
    measured = (raw.mean(-1).abs() / raw.std(-1)).min().item()
    return measured, errs


@pytest.mark.parametrize("ratio", [1, 10, 100])
def test_gn_large_mean_split(dev, ratio):
    """GroupNorm statistics are E[x^2] - mean^2 in double from fp32 per-warp partial sums of 256 values, so the relative
    variance error can grow like ~1e-7 (r^2 + 1) with r = |mean| / std.  Measured on head conv 4 (64 x 64, B = 3) in split
    mode, GroupNorm + GELU output error 7.9e-6 / 6.7e-6 / 2.0e-5 at r = 1 / 10 / 100 (1.5e-5 at r = 30; the conv output
    itself stays at 9e-6 - 1.0e-5): the split-mode bar of 4e-5 holds up to r = 100, the largest ratio measured.  The bf16
    mode stays at 4.0e-3 - 4.6e-3 over the same range."""
    measured, errs = gn_ratio_errors("bf16x3", ratio)
    assert 0.5 * ratio < measured < 2 * ratio, measured
    _assert_bars(errs, "bf16x3")
