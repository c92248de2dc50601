"""The ConvNeXt backbone one stage at a time (gdrn_model_run_stage: the forward's own stage functions, plans and kernels)
against float64 torch references of the same op, in both precision modes, for convnext_base and convnext_tiny (whose
stage 0 stores its 96 channels 128 wide: 32 zero pad channels through the stem LayerNorm, the stage-0 blocks and down1).

Reference per mode:
  * bf16x3: the fp64 op on the fp32 input and the fp32 weights.
  * bf16:   the fp64 op with the GEMM weights (stem_0, downsample.1, mlp.fc1, mlp.fc2) rounded to bf16; depthwise taps,
            biases, LayerNorm affines and gamma stay fp32, as the kernels read them.  The stem's input is rounded to bf16
            too: the stem GEMM reads the image as a bf16 operand in this mode.  The residual stream is fp32 in both modes.

Quantities: "stem" is the stem output (LayerNorm in the GEMM epilogue, fp32), "operand" the GEMM A operand the
LayerNorm kernels write (ln_patchify2 for down<s>, the depthwise conv + LayerNorm for block<s>_<i>; decoded hi + lo),
"down" / "block" the fp32 stage outputs.  Errors are max |got - ref| / max(1, max |ref|).  Each bar is at most 4x the
largest error measured on an H100 (80GB HBM3, 400 W power limit) over all cases of the quantity; BARS lists that maximum
and where it occurred.

Depthwise kernel per (stage, B) (launch_dwconv_ln; _dw_kernel below restates the rule and
test_dwconv_kernel_coverage checks that every kernel is reached):
  * ping-pong kernel when B * (H/8) * (W/16) >= 32: stage 0 at every B, stage 1 at B = 5, 64, stage 2 at B = 64;
  * 16x8x64 cluster kernel: stage 1 at B = 1, 3, stage 2 at B = 1, 3, 5;
  * 8x8x128 cluster kernel: stage 3 (8 x 8 maps) at every B.
MLP paths: convnext_base stage 0 takes the fused kernel of its mode (mlp_fused / mlp_fused_x3); every other block,
including convnext_tiny's stage 0 (96 real of 128 stored channels), the unfused fc1-GELU / fc2-residual GEMMs.
test_block0_mlp_paths runs base stage 0 with the fused kernels disabled and with the fp32 GELU forms.

Inputs: every image carries its own offset (a read from a neighbouring image shows), the mean is non-zero, the outermost
3 rows and columns (the depthwise halo; they include the outermost 2x2 patch rows and columns) carry 3x the energy (the
stem input: its outermost 4-pixel patch rows and columns), and pad channels are zero.  Weights are seeded from a state
dict owned by this file, every block differently, at the scale of a trained network with gamma in [0.1, 1].
"""
import functools
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import gdrn_model_oracle as O

MODES = ("bf16x3", "bf16")
BATCHES = (1, 3, 5, 64)
ARCHS = ("convnext_base", "convnext_tiny")
GEMM_WEIGHTS = ("stem_0.weight", "downsample.1.weight", "mlp.fc1.weight", "mlp.fc2.weight")

# (quantity, mode) -> bar, with the largest error measured over all cases of the quantity (H100 80GB HBM3, 400 W power
# limit) and where it occurred.
BARS = {
    ("stem", "bf16x3"): 2.5e-5,      # 6.32e-6  base B=64
    ("stem", "bf16"): 1.2e-6,        # 3.08e-7  base B=3 (bf16 operands of the reference too: fp32 accumulation only)
    ("operand", "bf16x3"): 2.2e-5,   # 5.73e-6  tiny down3 B=3 (hi + lo of the LayerNorm output, 2^-17)
    ("operand", "bf16"): 1.4e-2,     # 3.59e-3  tiny block2_0 B=64 (bf16 rounding of the LayerNorm output, 2^-9)
    ("down", "bf16x3"): 3.8e-5,      # 9.51e-6  base down3 B=3
    ("down", "bf16"): 7.9e-3,        # 1.98e-3  tiny down3 B=64
    ("block", "bf16x3"): 2.2e-5,     # 5.46e-6  base block3_0 B=64
    ("block", "bf16"): 3.4e-3,       # 8.61e-4  base block0_0 B=5 (fused and unfused MLP alike)
}

# The same quantities with |mean| / std = 1, 10, 100 in the stem, block0_0 and down1 LayerNorms (B = 3, both archs).
# Measured maximum over the three ratios after masking the pad channels out of the centred pass, and (in brackets) with
# the pad-corrected form the kernels used before, (C - c_real) * mean^2 subtracted from a sum over all stored channels.
LARGE_MEAN_BARS = {
    ("stem", "bf16x3"): 1.2e-4,      # 3.07e-5  base r=100 (before: 2.18e-3 tiny r=100)
    ("stem", "bf16"): 1.5e-4,        # 3.80e-5  tiny r=100 (before: 2.96e-3 tiny r=100)
    ("operand", "bf16x3"): 4.7e-5,   # 1.18e-5  base block0_0 r=100 (before: 2.06e-4 tiny down1 r=100)
    ("operand", "bf16"): 1.1e-2,     # 2.78e-3  base block0_0 r=100
    ("down", "bf16x3"): 3.5e-5,      # 8.81e-6  tiny down1 r=100 (before: 1.50e-4 tiny down1 r=100)
    ("down", "bf16"): 7.6e-3,        # 1.91e-3  base down1 r=100
    ("block", "bf16x3"): 1.8e-5,     # 4.48e-6  base block0_0 r=1 (before: 4.34e-5 tiny block0_0 r=100)
    ("block", "bf16"): 6.9e-3,       # 1.72e-3  tiny block0_0 r=1
}


def _arch(arch):
    depths, dims = O.CONVNEXT_ARCH[arch]
    return depths, dims, [(d + 63) // 64 * 64 for d in dims]


def _stages(arch):
    depths, _, _ = _arch(arch)
    return (["stem"] + [f"down{s}" for s in (1, 2, 3)] + [f"block{s}_0" for s in range(4)]
            + [f"block2_{depths[2] - 1}"])


CASES = [(a, st) for a in ARCHS for st in _stages(a)]


def _dw_kernel(s, B):
    """The depthwise kernel launch_dwconv_ln picks for stage s at batch B (variant -1, as the forward calls it)."""
    r = 64 >> s
    if B * (r // 8) * (r // 16) >= 32:
        return "ping-pong"
    return "cluster 16x8x64" if r % 16 == 0 else "cluster 8x8x128"


def _err(got, ref):
    got, ref = got.double(), ref.double()
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item())


def _assert_bars(errs, mode, bars=BARS):
    for (what, q), e in errs.items():
        assert e <= bars[(q, mode)], (what, q, mode, e, bars[(q, mode)])


# ------------------------------------------------------------------------------------------------ fixtures
def _state_dict(arch, seed=0):
    """Seeded backbone weights at the scale of a trained network: He-initialised convs and linears, depthwise taps of
    std 1/7, LayerNorm affines near (1, 0), biases of std 0.1, gamma uniform in [0.1, 1].  One generator runs through
    the keys in order, so every block gets its own weights.  The head is zero (no backbone stage reads it)."""
    from gdrnpp_bop2022_b200.synthetic import state_dict_shapes

    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, s in state_dict_shapes(arch, 21).items():
        if not k.startswith("backbone."):
            sd[k] = torch.zeros(s)
        elif k.endswith("conv_dw.weight"):
            sd[k] = torch.randn(s, generator=g) / 7.0
        elif k.endswith("mlp.fc2.weight"):
            sd[k] = torch.randn(s, generator=g) * (1.0 / s[1]) ** 0.5
        elif len(s) >= 2:   # stem_0 / downsample.1 convs, fc1
            sd[k] = torch.randn(s, generator=g) * (2.0 / math.prod(s[1:])) ** 0.5
        elif k.endswith("gamma"):
            sd[k] = 0.1 + 0.9 * torch.rand(s, generator=g)
        elif k.endswith("weight"):   # LayerNorm affine
            sd[k] = 1.0 + 0.2 * torch.randn(s, generator=g)
        else:
            sd[k] = 0.1 * torch.randn(s, generator=g)
    return sd


def _ref_sd(sd, mode):
    dev = torch.device("cuda:0")
    ref = {}
    for k, v in sd.items():
        if not k.startswith("backbone."):
            continue
        if mode == "bf16" and k.endswith(GEMM_WEIGHTS):
            v = v.bfloat16().float()
        ref[k] = v.double().to(dev)
    return ref


def _model(arch, mode, sd, max_batch=64):
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg

    model = GDRN_DoubleMask(default_cfg(arch=arch), arch=arch, max_batch=max_batch, precision=mode)
    model.load_state_dict(sd)
    return model


@functools.lru_cache(maxsize=None)
def _setup(arch, mode):
    """(model, fp64 reference state dict) of one arch and precision mode."""
    sd = _state_dict(arch)
    return _model(arch, mode, sd), _ref_sd(sd, mode)


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _setup.cache_clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _input(shape, seed, c_real, band=3, gain=3.0):
    """NHWC [B,H,W,C]: unit noise, `gain` x in the outermost `band` rows / columns, mean 0.3 plus a per-image offset,
    zero channels from c_real on."""
    B, H, W, C = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g)
    e = torch.ones(H, W)
    e[:band, :] = e[-band:, :] = e[:, :band] = e[:, -band:] = gain
    off = 0.3 + 0.2 * ((torch.arange(B) * 5) % 7 - 3).float()
    x = x * e[None, :, :, None] + off[:, None, None, None]
    x[..., c_real:] = 0.0
    return x


def _image(B, seed):
    """roi_img [B,3,256,256]: values in [0, 1) with a per-image offset, 3x the spread in the outermost 4-pixel patches."""
    x = _input((B, 256, 256, 3), seed, 3, band=4).permute(0, 3, 1, 2).contiguous()
    return x * 0.25 + 0.5


def _run_twice(model, stage, x, want_raw):
    """Runs a stage twice on the same input: both outputs must be bit-identical."""
    a = model.run_stage(stage, x, want_raw=want_raw)
    b = model.run_stage(stage, x, want_raw=want_raw)
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), (stage, k)
    return a


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _patch_rows(n):
    """LayerNorm2d output NCHW [B,C,2r,2r] -> the downsample GEMM's patch rows [B,r,r,2(dy),2(dx),C]."""
    B, C, H, W = n.shape
    return n.permute(0, 2, 3, 1).reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5)


# ------------------------------------------------------------------------------------------------ stages
def stage_errors(arch, stage, mode, B, model=None, sd=None, x=None):
    """{(stage, quantity): error} of one backbone stage; also checks pad channels and run-to-run bit identity."""
    if model is None:
        model, sd = _setup(arch, mode)
    depths, dims, cp = _arch(arch)
    seed = 7 * B + sum(map(ord, stage))
    with torch.no_grad():
        if stage == "stem":
            if x is None:
                x = _image(B, seed)
            res = _run_twice(model, stage, x.cuda(), want_raw=False)
            xr = (x.bfloat16().float() if mode == "bf16" else x).double().cuda()
            ref = O.convnext_stem(sd, xr)
            out = res["out"]
            if cp[0] > dims[0]:
                assert out[..., dims[0]:].abs().max().item() == 0.0
            return {(stage, "stem"): _err(_nchw(out[..., :dims[0]]), ref)}
        if stage.startswith("down"):
            s = int(stage[4:])
            r = 64 >> s
            if x is None:
                x = _input((B, 2 * r, 2 * r, cp[s - 1]), seed, dims[s - 1])
            res = _run_twice(model, stage, x.cuda(), want_raw=True)
            ref, n = O.convnext_downsample(sd, _nchw(x[..., :dims[s - 1]].double().cuda()), s, return_norm=True)
            op = res["raw"].reshape(B, r, r, 2, 2, cp[s - 1])
            if cp[s - 1] > dims[s - 1]:
                assert op[..., dims[s - 1]:].abs().max().item() == 0.0     # pad slots of every patch position
            return {(stage, "operand"): _err(op[..., :dims[s - 1]], _patch_rows(n)),
                    (stage, "down"): _err(_nchw(res["out"]), ref)}
        s, i = (int(v) for v in stage[5:].split("_"))
        r = 64 >> s
        if x is None:
            x = _input((B, r, r, cp[s]), seed, dims[s])
        res = _run_twice(model, stage, x.cuda(), want_raw=True)
        ref, n = O.convnext_block(sd, _nchw(x[..., :dims[s]].double().cuda()), s, i, return_norm=True)
        if cp[s] > dims[s]:
            assert res["out"][..., dims[s]:].abs().max().item() == 0.0
            assert res["raw"][..., dims[s]:].abs().max().item() == 0.0
        return {(stage, "operand"): _err(res["raw"][..., :dims[s]], n),
                (stage, "block"): _err(_nchw(res["out"][..., :dims[s]]), ref)}


@pytest.mark.gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("arch,stage", CASES)
def test_backbone_stage_vs_fp64(dev, arch, stage, mode, B):
    """Stem (GEMM + EPI_BIAS_LN), downsamples (ln_patchify2 + GEMM) and blocks (depthwise 7x7 + LayerNorm + MLP) against
    fp64; block2_26 / block2_8 is the last stage-2 block (per-block weight indexing)."""
    _assert_bars(stage_errors(arch, stage, mode, B), mode)


@pytest.mark.gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("mode,env", [("bf16x3", {"GDRN_MLP_FUSED_X3": "0"}), ("bf16", {"GDRN_MLP_FUSED": "0"}),
                                      ("bf16", {"GDRN_GELU_MODE": "0"}), ("bf16", {"GDRN_GELU_MODE": "2"})],
                         ids=["x3-unfused", "bf16-unfused", "bf16-gelu0", "bf16-gelu2"])
def test_block0_mlp_paths(dev, monkeypatch, mode, env, B):
    """convnext_base block0_0 through the unfused fc1-GELU / fc2-residual GEMMs (the fused kernels disabled) and, in bf16
    mode, with the fp32 GELU forms of the fc1 epilogue (0: ex2 / rcp, 2: tanh.approx; both leave the fused kernel)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    _, sd = _setup("convnext_base", mode)
    model = _model("convnext_base", mode, _state_dict("convnext_base"), max_batch=B)
    try:
        _assert_bars(stage_errors("convnext_base", "block0_0", mode, B, model=model, sd=sd), mode)
    finally:
        del model
        torch.cuda.empty_cache()


def test_dwconv_kernel_coverage():
    """The (stage, B) cases of test_backbone_stage_vs_fp64 reach all three depthwise kernels."""
    hit = {_dw_kernel(s, B) for s in range(4) for B in BATCHES}
    assert hit == {"ping-pong", "cluster 16x8x64", "cluster 8x8x128"}, hit
    assert {_dw_kernel(s, B) for s in (1, 2) for B in BATCHES} == {"ping-pong", "cluster 16x8x64"}


# ------------------------------------------------------------------------------------------------ LayerNorm, large mean
def _ratio_state_dict(arch, ratio):
    """Weights that put |mean| / std ~ ratio into the stem LayerNorm and into block0_0's LayerNorm.
      * stem: the bias is the common offset 1.41 * ratio.  The stem conv spreads a [0, 1) image patch over the channels
        with std ~0.85, so the median ratio comes out at ~1.65 x ratio.
      * block0_0: every channel's 49 taps sum to 1 and its bias is 0, so an input DC offset of 0.15 * ratio passes
        through as the mean, over a spread of ~0.15.
    The downsample takes its ratio from the input's DC offset alone."""
    sd = _state_dict(arch)
    g = torch.Generator().manual_seed(900)
    b = sd["backbone.stem_0.bias"]
    sd["backbone.stem_0.bias"] = 1.41 * ratio + 0.1 * torch.randn(b.shape, generator=g)
    w = sd["backbone.stages_0.blocks.0.conv_dw.weight"]
    t = 1.0 + 0.3 * torch.randn(w.shape, generator=g)
    sd["backbone.stages_0.blocks.0.conv_dw.weight"] = (t - t.mean(dim=(2, 3), keepdim=True) + 1.0) / 49.0
    sd["backbone.stages_0.blocks.0.conv_dw.bias"] = torch.zeros_like(sd["backbone.stages_0.blocks.0.conv_dw.bias"])
    return sd


def _median_ratio(y):
    """Median over pixels of |mean| / std over the channels of NCHW y."""
    return (y.mean(dim=1).abs() / y.std(dim=1)).median().item()


def large_mean_errors(arch, mode, ratio, B=3):
    """{(stage, quantity): error} and the measured median |mean| / std per LayerNorm, for stem, block0_0 and down1."""
    _, dims, cp = _arch(arch)
    sd = _ratio_state_dict(arch, ratio)
    ref_sd = _ref_sd(sd, mode)
    model = _model(arch, mode, sd, max_batch=B)
    errs, measured = {}, {}
    g = torch.Generator().manual_seed(950 + int(ratio))
    with torch.no_grad():
        img = torch.rand(B, 3, 256, 256, generator=g)
        errs.update(stage_errors(arch, "stem", mode, B, model=model, sd=ref_sd, x=img))
        xr = (img.bfloat16().float() if mode == "bf16" else img).double().cuda()
        measured["stem"] = _median_ratio(F.conv2d(xr, ref_sd["backbone.stem_0.weight"], ref_sd["backbone.stem_0.bias"],
                                                  stride=4))
        for stage, dc in (("block0_0", 0.15 * ratio), ("down1", 1.0 * ratio)):
            x = torch.randn(B, 64, 64, cp[0], generator=g) + dc
            x[..., dims[0]:] = 0.0
            errs.update(stage_errors(arch, stage, mode, B, model=model, sd=ref_sd, x=x))
            xd = _nchw(x[..., :dims[0]].double().cuda())
            if stage == "block0_0":
                p = "backbone.stages_0.blocks.0."
                xd = F.conv2d(xd, ref_sd[p + "conv_dw.weight"], ref_sd[p + "conv_dw.bias"], padding=3, groups=dims[0])
            measured[stage] = _median_ratio(xd)
    del model
    torch.cuda.empty_cache()
    return errs, measured


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [1, 10, 100])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("arch", ARCHS)
def test_ln_large_mean(dev, arch, mode, ratio):
    """The LayerNorms that see zero pad channels on convnext_tiny at |mean| / std ~ 1, 10, 100 per pixel: the stem
    epilogue, the depthwise ping-pong kernel (stage 0 always takes it) and ln_patchify2; convnext_base runs the same
    LayerNorms without pad channels.  Taking the centred sum of squares over all stored channels and subtracting the pad
    channels' (C - c_real) * mean^2 afterwards cancels here: at r = 100 the split-mode stem output was off by 2.2e-3 and
    the down1 operand by 2.1e-4 (LARGE_MEAN_BARS).  The kernels now mask the pad channels out of the centred pass."""
    errs, measured = large_mean_errors(arch, mode, ratio)
    for k, v in measured.items():
        assert 0.5 * ratio < v < 2 * ratio, (k, v)
    _assert_bars(errs, mode, LARGE_MEAN_BARS)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("arch", ARCHS)
def test_ln_mean_1000_report(dev, arch, mode):
    """|mean| / std ~ 1000, reported without a bar (fp32 statistics lose about log10(ratio^2) digits there)."""
    errs, measured = large_mean_errors(arch, mode, 1000)
    print(f"\n{arch} {mode} |mean|/std=1000: measured {measured}, errors {errs}")
    assert all(math.isfinite(e) for e in errs.values()), errs


# ------------------------------------------------------------------------------------------------ chain = forward
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("arch", ARCHS)
def test_stage_chain_is_forward(dev, arch, mode):
    """stem -> blocks -> downs through run_stage reproduces gdrn_model_forward's backbone output bit for bit: the stages
    are the forward's own code."""
    from gdrnpp_bop2022_b200.synthetic import make_batch

    model, _ = _setup(arch, mode)
    depths, _, cp = _arch(arch)
    B = 3
    batch = {k: v.cuda() for k, v in make_batch(B=B, seed=5).items()}
    img = _image(B, 77).cuda()
    model(img, roi_classes=batch["roi_classes"], roi_coord_2d=batch["roi_coord_2d"], roi_cams=batch["roi_cams"],
          roi_centers=batch["roi_centers"], roi_whs=batch["roi_whs"], roi_extents=batch["roi_extents"],
          resize_ratios=batch["resize_ratios"])
    torch.cuda.synchronize()
    fwd = model.debug_read("stage3_x", B, B * 64 * cp[3]).reshape(B, 8, 8, cp[3]).clone()
    x = model.run_stage("stem", img)["out"]
    for s in range(4):
        if s > 0:
            x = model.run_stage(f"down{s}", x)["out"]
        for i in range(depths[s]):
            x = model.run_stage(f"block{s}_{i}", x)["out"]
    torch.cuda.synchronize()
    assert torch.equal(x, fwd)


# ------------------------------------------------------------------------------------------------ stage names
@pytest.mark.gpu
def test_stage_names_rejected(dev):
    """gdrn_model_run_stage's parser: out-of-range stage / block indices (two-digit block indices of stage 2 accepted up
    to depth - 1), malformed names and GroupNorm sums / conv outputs a backbone stage does not have."""
    from gdrnpp_bop2022_b200 import _lib

    model, _ = _setup("convnext_tiny", "bf16x3")
    B = 1
    x = torch.zeros(B, 3, 256, 256, device="cuda")
    model.run_stage("stem", x)   # creates the engine and workspace
    ws = model._get_workspace(B, x.device)
    buf = torch.empty(B * 256 * 256 * 128, device="cuda")
    stats = torch.empty(10 * B * 64, dtype=torch.float64, device="cuda")

    def rc(stage, raw=None, gn=None):
        return _lib.lib().gdrn_model_run_stage(model._handle, stage.encode(), B, _lib.ptr(buf), _lib.ptr(buf), raw, gn,
                                               None, None, None, None, _lib.ptr(ws), ws.numel(), _lib.current_stream())

    for bad in ("block2_9", "block0_3", "block3_3", "block4_0", "block2_08", "block2_", "block2", "block_1", "block1_-1",
                "down0", "down4", "down1x", "stem1", "head_conv6", "pnp_conv3", "block22_0", "block2_1234567"):
        assert rc(bad) != 0, bad
    assert rc("block2_8") == 0 and rc("down3") == 0
    assert rc("stem", raw=_lib.ptr(buf)) != 0
    for st in ("stem", "down1", "block0_0"):
        assert rc(st, gn=_lib.ptr(stats)) != 0, st
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        model.run_stage("block2_9", torch.zeros(B, 16, 16, 384, device="cuda"))


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("arch", ARCHS)
def test_oracle_stages_compose_to_features(arch):
    """convnext_stem -> (convnext_downsample) -> convnext_block, with the LayerNorm outputs requested, equals
    convnext_features in fp64; the downsample's returned LayerNorm output is the LayerNorm of its input."""
    sd = {k: v.double() for k, v in _state_dict(arch).items() if k.startswith("backbone.")}
    depths, _, _ = _arch(arch)
    g = torch.Generator().manual_seed(3)
    img = torch.rand(2, 3, 64, 64, generator=g, dtype=torch.float64)
    with torch.no_grad():
        x = O.convnext_stem(sd, img)
        for s in range(4):
            if s > 0:
                y, n = O.convnext_downsample(sd, x, s, return_norm=True)
                p = f"backbone.stages_{s}.downsample.0."
                z = F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), sd[p + "weight"], sd[p + "bias"], 1e-6)
                assert torch.equal(n, z.permute(0, 3, 1, 2))
                x = y
            for i in range(depths[s]):
                y, n = O.convnext_block(sd, x, s, i, return_norm=True)
                assert torch.equal(y, O.convnext_block(sd, x, s, i))
                assert n.shape == x.permute(0, 2, 3, 1).shape
                x = y
        assert torch.equal(x, O.convnext_features(sd, img, arch))
