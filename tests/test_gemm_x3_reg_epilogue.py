"""The split-bf16 GEMM's register epilogue (gdrn_gemm_x3 on plain rank-2 rows: EPI_STORE, EPI_GELU and EPI_RESID run
straight from the wgmma fragments, and the operand ring is 3 stages deep at BLOCK_N 128, 4 at BLOCK_N 64).

- Ring wrap at those depths: K = 64, 192, 256, 320, 448 gives 1, 3, 4, 5 and 7 k-chunks; M is ragged and large enough that
  every persistent CTA runs several tiles, and N = 192 leaves the last 128-wide tile half empty (columns >= N masked).
  Checked against an fp64 product, for run-to-run identical bits and for untouched canary rows behind the matrix.
- Bit identity: SHA-256 digests of the outputs at the stage-1..3 MLP, downsample and small-batch shapes, recorded from
  the accumulator-tile epilogue by tools/make_golden_gemm_x3.py (tests/golden/gemm_x3_digests.json).  The mainloop and
  the per-element operations are the same, so every byte must be too."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden_gemm_x3 as G  # noqa: E402

pytestmark = pytest.mark.gpu

M_WRAP = 128 * 132 * 3 + 37   # ~6 tiles per CTA on 132 SMs at N = 192, BLOCK_N 128; ragged last tile
N_WRAP = 192


def _split_bf16(t):
    hi = t.bfloat16()
    lo = (t - hi.float()).bfloat16()
    return torch.cat([hi, lo], dim=1).contiguous()


@pytest.mark.parametrize("epi", [0, 1, 2])
@pytest.mark.parametrize("K", [64, 192, 256, 320, 448])
@pytest.mark.parametrize("bn", [64, 128])
def test_gemm_x3_reg_ring_wraps(dev, lib, bn, K, epi):
    from gdrnpp_bop2022_b200 import _lib as L

    M, N = M_WRAP, N_WRAP
    g = torch.Generator().manual_seed(7000 + 1000 * bn + 10 * K + epi)
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev)
    W = (torch.randn(N, K, generator=g) / np.sqrt(K)).to(dev)
    bias, gamma = torch.randn(N, generator=g).to(dev), torch.rand(N, generator=g).to(dev)
    x = torch.randn(M, N, generator=g).to(dev)
    ref = A.double() @ W.double().t() + bias.double()
    if epi == 1:
        ref = torch.nn.functional.gelu(ref)
    if epi == 2:
        ref = x.double() + gamma.double() * ref
    A2, W2 = _split_bf16(A), _split_bf16(W)
    outs = []
    for _ in range(2):
        if epi == 1:
            out = torch.full((M + 64, 2 * N), float("nan"), dtype=torch.bfloat16, device=dev)
        else:
            out = torch.full((M + 64, N), 7.0, dtype=torch.float32, device=dev)   # canary rows behind the matrix
            if epi == 2:
                out[:M] = x
        L.check(lib.gdrn_gemm_x3(L.ptr(A2), L.ptr(W2), L.ptr(bias), L.ptr(gamma), L.ptr(out), L.ptr(out), M, N, K, epi, bn,
                                 L.current_stream()), "gemm_x3")
        torch.cuda.synchronize()
        if epi == 1:
            assert torch.isnan(out[M:].float()).all()
        else:
            assert torch.equal(out[M:], torch.full((64, N), 7.0, device=dev))
        outs.append(out[:M].clone())
    assert torch.equal(outs[0], outs[1])
    got = outs[0][:, :N].double() + outs[0][:, N:].double() if epi == 1 else outs[0].double()
    err = (got - ref).abs().max().item()
    assert err < 4e-5 * max(1.0, ref.abs().max().item()), err


def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "gemm_x3_digests.json")) as f:
        return {c["name"]: c for c in json.load(f)["cases"]}


@pytest.mark.parametrize("case", G.CASES, ids=[c[0] for c in G.CASES])
def test_gemm_x3_bits_match_golden(dev, lib, case):
    rec = _golden()[case[0]]
    assert (rec["M"], rec["N"], rec["K"], rec["epi"], rec["block_n"]) == tuple(case[1:])
    assert G.digest_case(lib, dev, case) == rec["sha256"]
