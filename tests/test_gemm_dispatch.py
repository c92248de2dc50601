"""Which implicit-GEMM kernel each GEMM call site of the GDRN forward runs, and whether an fp64 test checks it there.

gdrn_gemm_kernels_launched() records the kernels the library launched since the last reset (one bit per instantiation of
gemm_tc_launch plus the two fused ConvNeXt MLP kernels; _lib.GEMM_KERNELS names them).  The dispatch map runs every stage
gdrn_model_run_stage accepts -- convnext_base's backbone, geometry head and Patch-PnP and convnext_tiny's backbone, one
block per stage plus the last stage-2 block, the stages the fp64 stage tests run -- at batches that straddle every tile-width
switch, in both precision modes and at the default environment, and records (arch, stage, B, mode) -> kernels.  The rules
behind it are spread out: pick_bn narrows 256 -> 128 -> 64 until a launch covers half a wave of SMs, the deconv takes
256-wide tiles (run as 128) only from 96 row tiles on (B >= 191), gemm_tc_launch folds 256 into 128 and picks the 32-wide
k-chunk ring for split-bf16 convolutions and the register epilogue for split-bf16 plain rows.

  (a) every stage runs (GDRN_OK) at every batch in both modes: a split-bf16 plan that matches no kernel is an error;
  (b) the map plus the stand-alone GEMM entries (gdrn_gemm_bf16, gdrn_gemm_x3, gdrn_mlp_fused_x3 at the (epi, block_n)
      of their tests) reach every kernel, or the kernel is listed in UNREACHED;
  (c) every (arch, stage, mode, kernel) of the map is also reached by a batch at which an fp64 test checks that stage
      (FP64_BATCHES): a dispatch change that sends a stage to a kernel no fp64 case runs it through fails here, naming the
      pair, until an fp64 case is added for it.

The fp64 cases this file adds: the deconv at B = 191 and 192 (128-wide GroupNorm-sum tiles: two images per 8x8 box, the
1 / 2 / 4-tap parity plans, the stride-2 gather store, GroupNorm sums split over two N tiles), and the bf16 GELU epilogue
in its erff form (GDRN_GELU_MODE=3).  The map itself computes no references; it is cheap.
"""
import functools
import os
import re

import pytest
import torch

import test_backbone_stages as BB
import test_head_stages as HS
from conftest import ROOT

MODES = ("bf16x3", "bf16")
ARCHS = ("convnext_base", "convnext_tiny")
HEAD = HS.HEAD_STAGES + ("out_conv", "pnp_conv0", "pnp_conv1", "pnp_conv2", "pnp_fc")

# The batches at which an fp64 test checks each stage, in both modes (restated from the parametrizations of
# test_backbone_stages.py::test_backbone_stage_vs_fp64, test_head_stages.py::test_head_stage_vs_fp64, test_out_conv_vs_fp64,
# test_pnp_conv_vs_fp64 and test_pnp_fc_vs_fp64, and from test_deconv_wide_tiles_vs_fp64 below;
# test_fp64_batches_restate_the_stage_tests keeps them in step).
_B4 = (1, 3, 5, 64)
WIDE_DECONV_BATCHES = (191, 192)     # ceil(B / 2) >= 96 row tiles: the deconv's 128-wide tiles; 191 leaves a half box
FP64_BATCHES = {
    **{("convnext_base", s): _B4 for s in ("stem", "down1", "down2", "down3", "block0_0", "block1_0", "block2_0",
                                           "block3_0", "block2_26")},
    **{("convnext_tiny", s): _B4 for s in ("stem", "down1", "down2", "down3", "block0_0", "block1_0", "block2_0",
                                           "block3_0", "block2_8")},
    ("convnext_base", "deconv"): _B4 + WIDE_DECONV_BATCHES,
    **{("convnext_base", f"head_conv{i}"): _B4 for i in range(6)},
    ("convnext_base", "out_conv"): _B4,
    **{("convnext_base", f"pnp_conv{i}"): _B4 for i in range(3)},
    ("convnext_base", "pnp_fc"): (1, 16, 17, 20, 64),
}

# Batches of the dispatch map: both sides of every width switch of convnext_base and convnext_tiny (pick_bn's half wave of
# 66 CTAs on 132 SMs; the deconv's 96 row tiles) and every fp64 batch.
MAP_BATCHES = tuple(sorted({1, 2, 3, 4, 5, 8, 9, 16, 17, 20, 33, 64, 96, 190, 191, 192, 256}
                           | {b for bs in FP64_BATCHES.values() for b in bs}))

# Kernels that neither the forward (at any batch of the map) nor a stand-alone GEMM test reaches.  Keep each with the
# reason; deleting one is a change of its own.
UNREACHED = {}

# Stand-alone entries at the (epi, block_n) their tests call them with -> the kernel each call must record.
# test_gpu_parity.py::test_gemm_vs_torch / test_gemm_residual_in_place / test_gemm_gelu_modes (and mode 3 below):
STANDALONE_BF16 = {(0, 128): "bf16 128 STORE bk64", (0, 256): "bf16 128 STORE bk64", (1, 256): "bf16 128 GELU bk64",
                   (2, 128): "bf16 128 RESID bk64", (2, 256): "bf16 128 RESID bk64", (1, 64): "bf16 64 GELU bk64",
                   (0, 16): "bf16 16 STORE bk64"}
# test_gpu_parity.py::test_gemm_x3_vs_fp64 / test_gemm_x3_residual_in_place, test_gemm_x3_ring.py, test_gemm_x3_reg_epilogue.py:
STANDALONE_X3 = {(e, bn): f"x3 {min(bn, 128)} {('STORE', 'GELU', 'RESID')[e]} bk64 reg"
                 for e in (0, 1, 2) for bn in (64, 128, 256)}


def _L():
    from gdrnpp_bop2022_b200 import _lib

    return _lib


# ------------------------------------------------------------------------------------------------ CPU
def test_kernel_names_follow_the_instantiation_table():
    """_lib.GEMM_KERNELS names the bits in the order of gemm_tc.cu's kGemmKernels table, then the two fused MLPs."""
    src = open(os.path.join(ROOT, "gdrnpp_bop2022_b200", "csrc", "gemm_tc.cu")).read()
    table = re.search(r"constexpr GemmKernelKey kGemmKernels\[\] = \{(.*?)\n\};", src, re.S).group(1)
    rows = re.findall(r"\{(\d+), EPI_(\w+), (true|false), (\d+), (true|false)\}", table)
    names = [f"{'x3' if x3 == 'true' else 'bf16'} {bn} {epi} bk{bk}{' reg' if reg == 'true' else ''}"
             for bn, epi, x3, bk, reg in rows]
    hdr = open(os.path.join(ROOT, "gdrnpp_bop2022_b200", "csrc", "gemm_tc.h")).read()
    n_tc = int(re.search(r"constexpr int GEMM_NUM_TC_KERNELS = (\d+);", hdr).group(1))
    assert len(names) == n_tc == 20
    assert tuple(names) + ("mlp_fused", "mlp_fused_x3") == _L().GEMM_KERNELS
    assert _L().gemm_kernel_names(0b101) == ["bf16 128 GELU bk64", "bf16 128 STORE bk64"]
    with pytest.raises(ValueError):
        _L().gemm_kernel_names(1 << len(_L().GEMM_KERNELS))


def _param_values(fn, name):
    for m in fn.pytestmark:
        if m.name == "parametrize" and m.args[0] == name:
            return tuple(m.args[1])
    raise AssertionError(f"{fn.__name__} has no parametrize({name!r})")


def test_fp64_batches_restate_the_stage_tests():
    """FP64_BATCHES lists exactly the (arch, stage, B) cases the fp64 stage tests run (both modes each)."""
    assert BB.MODES == HS.MODES == MODES
    want = {}
    for arch in BB.ARCHS:
        for stage in BB._stages(arch):
            want[(arch, stage)] = BB.BATCHES
    for stage in HS.HEAD_STAGES:
        want[("convnext_base", stage)] = HS.BATCHES
    want[("convnext_base", "deconv")] = HS.BATCHES + WIDE_DECONV_BATCHES
    want[("convnext_base", "out_conv")] = _param_values(HS.test_out_conv_vs_fp64, "B")
    for i in _param_values(HS.test_pnp_conv_vs_fp64, "i"):
        want[("convnext_base", f"pnp_conv{i}")] = _param_values(HS.test_pnp_conv_vs_fp64, "B")
    want[("convnext_base", "pnp_fc")] = _param_values(HS.test_pnp_fc_vs_fp64, "B")
    assert FP64_BATCHES == want
    assert BB.ARCHS == ARCHS
    assert set(FP64_BATCHES) == {(a, s) for a in ARCHS for s in BB._stages(a)} | {("convnext_base", s) for s in HEAD}


# ------------------------------------------------------------------------------------------------ dispatch map (GPU)
def _stage_args(arch, stage, B, dev):
    """Zero input of `stage` at batch B (dispatch depends on shapes only) and the extra run_stage arguments."""
    _, _, cp = BB._arch(arch)
    kw = {}
    if stage == "stem":
        shape = (B, 3, 256, 256)
    elif stage.startswith("down"):
        s = int(stage[4:])
        shape = (B, 2 * (64 >> s), 2 * (64 >> s), cp[s - 1])
    elif stage.startswith("block"):
        s = int(stage[5])
        shape = (B, 64 >> s, 64 >> s, cp[s])
    elif stage == "deconv":
        shape = (B, 8, 8, cp[3])
    elif stage.startswith("head_conv"):
        h = 16 << (int(stage[-1]) // 2)
        shape = (B, h, h, 256)
    elif stage == "out_conv":
        shape = (B, 64, 64, 256)
        kw = dict(roi_classes=torch.zeros(B, dtype=torch.int64, device=dev),
                  roi_extents=torch.full((B, 3), 0.1, device=dev), roi_coord_2d=torch.zeros(B, 2, 64, 64, device=dev))
    elif stage.startswith("pnp_conv"):
        r = 64 >> int(stage[-1])
        shape = (B, r, r, 128)
    else:
        assert stage == "pnp_fc", stage
        shape = (B, 8, 8, 128)
    return torch.zeros(shape, device=dev), kw


@functools.lru_cache(maxsize=None)
def _dispatch_map():
    """({(arch, stage, B, mode): frozenset of kernel names}, {(arch, stage, B, mode): error of a failed call})."""
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg

    L = _L()
    lib = L.lib()
    dev = torch.device("cuda:0")
    kmap, failed = {}, {}
    for arch in ARCHS:
        stages = [s for a, s in FP64_BATCHES if a == arch]
        for mode in MODES:
            # zero weights: which kernel runs depends on the shapes alone
            model = GDRN_DoubleMask(default_cfg(arch=arch), arch=arch, max_batch=max(MAP_BATCHES), precision=mode)
            for stage in stages:
                for B in MAP_BATCHES:
                    x, kw = _stage_args(arch, stage, B, dev)
                    lib.gdrn_gemm_kernels_launched(1)
                    try:
                        model.run_stage(stage, x, **kw)
                        torch.cuda.synchronize()
                    except L.GdrnError as e:
                        failed[(arch, stage, B, mode)] = str(e)
                    kmap[(arch, stage, B, mode)] = frozenset(L.gemm_kernel_names(lib.gdrn_gemm_kernels_launched(1)))
                    del x, kw
            del model
            torch.cuda.empty_cache()
    return kmap, failed


def _format_map(kmap):
    """One line per (arch, stage, mode): the kernels per run of consecutive map batches that take the same ones."""
    lines = []
    for arch, stage in FP64_BATCHES:
        for mode in MODES:
            runs = []
            for B in MAP_BATCHES:
                ks = kmap[(arch, stage, B, mode)]
                if runs and runs[-1][2] == ks:
                    runs[-1][1] = B
                else:
                    runs.append([B, B, ks])
            parts = [f"B {b0}{'' if b0 == b1 else f'-{b1}'}: {', '.join(sorted(ks)) or '-'}" for b0, b1, ks in runs]
            lines.append(f"{arch} {stage} {mode}: " + "; ".join(parts))
    return "\n".join(lines)


@pytest.mark.gpu
def test_every_stage_dispatches_at_every_batch(dev):
    """(a) Every stage returns GDRN_OK at every batch of the map, in both modes, and every GEMM stage launches at least
    one kernel (pnp_fc in split-bf16 mode runs the fp32 CUDA-core FC stack, no GEMM kernel).  Prints the map."""
    kmap, failed = _dispatch_map()
    print("\n(arch, stage, B, mode) -> kernels\n" + _format_map(kmap))
    assert not failed, failed
    empty = [k for k, ks in kmap.items() if not ks and not (k[1] == "pnp_fc" and k[3] == "bf16x3")]
    assert not empty, empty
    assert all(not ks for k, ks in kmap.items() if k[1] == "pnp_fc" and k[3] == "bf16x3")


def _standalone_kernels(dev):
    """{call: kernels recorded} for one small call of each stand-alone (entry, epi, block_n) of STANDALONE_*."""
    L = _L()
    lib = L.lib()
    st = L.current_stream()
    M, N, K = 256, 128, 64
    A, W = torch.zeros(M, 2 * K, dtype=torch.bfloat16, device=dev), torch.zeros(N, 2 * K, dtype=torch.bfloat16, device=dev)
    vec, x = torch.zeros(4 * N, device=dev), torch.zeros(M, N, device=dev)
    out = torch.zeros(M, 2 * N, device=dev)       # room for every output form (fp32 [M,N], split bf16 [M,2N])
    rec = {}
    for (epi, bn) in STANDALONE_BF16:
        lib.gdrn_gemm_kernels_launched(1)
        L.check(lib.gdrn_gemm_bf16(L.ptr(A), L.ptr(W), L.ptr(vec), L.ptr(vec), L.ptr(x), L.ptr(out), M, N, K, epi, 1, bn,
                                   st), "gemm_bf16")
        rec[("bf16", epi, bn)] = set(L.gemm_kernel_names(lib.gdrn_gemm_kernels_launched(1)))
    for (epi, bn) in STANDALONE_X3:
        lib.gdrn_gemm_kernels_launched(1)
        L.check(lib.gdrn_gemm_x3(L.ptr(A), L.ptr(W), L.ptr(vec), L.ptr(vec), L.ptr(out), L.ptr(out), M, N, K, epi, bn, st),
                "gemm_x3")
        rec[("x3", epi, bn)] = set(L.gemm_kernel_names(lib.gdrn_gemm_kernels_launched(1)))
    C = 128
    a2, w1 = torch.zeros(M, 2 * C, dtype=torch.bfloat16, device=dev), torch.zeros(4 * C, 2 * C, dtype=torch.bfloat16, device=dev)
    w2 = torch.zeros(C, 8 * C, dtype=torch.bfloat16, device=dev)
    lib.gdrn_gemm_kernels_launched(1)
    L.check(lib.gdrn_mlp_fused_x3(L.ptr(a2), L.ptr(w1), L.ptr(vec), L.ptr(w2), L.ptr(vec), L.ptr(vec), L.ptr(x), M, C, st),
            "mlp_fused_x3")
    rec[("mlp_fused_x3",)] = set(L.gemm_kernel_names(lib.gdrn_gemm_kernels_launched(1)))
    torch.cuda.synchronize()
    return rec


@pytest.mark.gpu
def test_standalone_entries_record_their_kernel(dev):
    """Each stand-alone call records exactly the kernel its (epi, block_n) selects; reading with reset = 0 keeps the
    record, reset != 0 clears it."""
    rec = _standalone_kernels(dev)
    want = {("bf16",) + k: {v} for k, v in STANDALONE_BF16.items()}
    want.update({("x3",) + k: {v} for k, v in STANDALONE_X3.items()})
    want[("mlp_fused_x3",)] = {"mlp_fused_x3"}
    assert rec == want
    L = _L()
    lib = L.lib()
    assert lib.gdrn_gemm_kernels_launched(0) == 0      # every call above read its record with reset
    M = 128
    A = torch.zeros(M, 64, dtype=torch.bfloat16, device=dev)
    out = torch.zeros(M, 16, device=dev)
    L.check(lib.gdrn_gemm_bf16(L.ptr(A), L.ptr(A), None, None, None, L.ptr(out), M, 16, 64, 0, 1, 16, L.current_stream()),
            "gemm_bf16")
    torch.cuda.synchronize()
    mask = lib.gdrn_gemm_kernels_launched(0)
    assert L.gemm_kernel_names(mask) == ["bf16 16 STORE bk64"]
    assert lib.gdrn_gemm_kernels_launched(1) == mask and lib.gdrn_gemm_kernels_launched(0) == 0


@pytest.mark.gpu
def test_every_kernel_is_reached(dev):
    """(b) The forward's stages and the stand-alone GEMM tests together reach every kernel not listed in UNREACHED, and
    nothing listed there is reached."""
    kmap, _ = _dispatch_map()
    forward = set().union(*kmap.values())
    standalone = set().union(*_standalone_kernels(dev).values())
    reached = forward | standalone
    known = set(_L().GEMM_KERNELS)
    assert reached <= known
    assert not (reached & set(UNREACHED)), sorted(reached & set(UNREACHED))
    assert reached | set(UNREACHED) == known, sorted(known - reached - set(UNREACHED))
    print("\nreached only by the stand-alone entries:", sorted(standalone - forward) or "-")


@pytest.mark.gpu
def test_every_dispatch_pair_has_an_fp64_case(dev):
    """(c) For every (arch, stage, mode) and every kernel the map sends it to at some batch, an fp64 test runs that stage
    at a batch (FP64_BATCHES) where it takes the same kernel."""
    kmap, _ = _dispatch_map()
    uncovered = []
    for (arch, stage), fp64_bs in FP64_BATCHES.items():
        for mode in MODES:
            checked = set().union(*(kmap[(arch, stage, B, mode)] for B in fp64_bs))
            for B in MAP_BATCHES:
                for k in sorted(kmap[(arch, stage, B, mode)] - checked):
                    uncovered.append(f"{arch} {stage} {mode}: {k} (first at B = {B})")
                    checked.add(k)
    assert not uncovered, "dispatch pairs no fp64 case checks:\n" + "\n".join(uncovered)


# ------------------------------------------------------------------------------------------------ fp64 cases
@pytest.mark.gpu
@pytest.mark.parametrize("B", WIDE_DECONV_BATCHES)
@pytest.mark.parametrize("mode", MODES)
def test_deconv_wide_tiles_vs_fp64(dev, mode, B):
    """The deconv at B >= 191 (ceil(B / 2) >= 96 row tiles): four parity GEMMs with 1 / 2 / 4 taps on 8x8 rank-4 boxes of
    two images each, 256 output channels as two 128-wide GroupNorm-sum tiles, stride-2 gather store.  Conv output,
    GroupNorm sums and GroupNorm + GELU output within the bars of test_head_stages.py; two runs bit-identical (GroupNorm
    sums: double atomics, to 1e-12); per-image offsets and 3x border energy in the input (test_head_stages._input).
    B = 191 leaves the second image of the last box beyond the batch.  The record shows the 128-wide kernel ran."""
    L = _L()
    lib = L.lib()
    lib.gdrn_gemm_kernels_launched(1)
    errs = HS.head_stage_errors("deconv", mode, B)
    want = "x3 128 GNSTATS bk32" if mode == "bf16x3" else "bf16 128 GNSTATS bk64"
    assert L.gemm_kernel_names(lib.gdrn_gemm_kernels_launched(1)) == [want]
    print(f"\ndeconv {mode} B={B}: " + ", ".join(f"{w} {q} {e:.3g}" for (w, q), e in errs.items()))
    HS._assert_bars(errs, mode)


@pytest.mark.gpu
def test_gemm_gelu_mode3_erf(dev, lib, monkeypatch):
    """The bf16 GELU epilogue's fourth form, erff (GDRN_GELU_MODE=3), vs erf-GELU of the same bf16 products at
    pre-activations up to ~ +-12 (test_gpu_parity.py::test_gemm_gelu_modes runs modes 0-2): within mode 0's bar, the
    bf16 rounding of the output (2^-8 of max(1, |ref|))."""
    L = _L()
    monkeypatch.setenv("GDRN_GELU_MODE", "3")
    g = torch.Generator().manual_seed(3)
    M, N, K = 512, 512, 256
    A = torch.randn(M, K, generator=g).to(dev).bfloat16()
    W = (torch.randn(N, K, generator=g) * (3.0 / K ** 0.5)).to(dev).bfloat16()
    bias = torch.randn(N, generator=g).to(dev)
    pre = A.double() @ W.double().t() + bias.double()
    ref = torch.nn.functional.gelu(pre)
    out = torch.empty((M, N), dtype=torch.bfloat16, device=dev)
    lib.gdrn_gemm_kernels_launched(1)
    L.check(lib.gdrn_gemm_bf16(L.ptr(A), L.ptr(W), L.ptr(bias), None, None, L.ptr(out), M, N, K, 1, 0, 256,
                               L.current_stream()), "gemm")
    torch.cuda.synchronize()
    assert L.gemm_kernel_names(lib.gdrn_gemm_kernels_launched(1)) == ["bf16 128 GELU bk64"]
    err = (out.double() - ref).abs()
    tol = 2.0 ** -8 * ref.abs().clamp_min(1.0)
    assert (err <= tol).all(), float((err - tol).max())
