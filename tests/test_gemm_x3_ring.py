"""Operand-ring bookkeeping of the split-bf16 GEMM kernel on plain rank-2 rows (gdrn_gemm_x3: 64-wide k-chunks, two ring
stages at BLOCK_N 128, three at BLOCK_N 64): chunk counts below the ring depth (K = 64: one chunk) and not a multiple of
it (K = 192, 320), and enough 128-row tiles that every persistent CTA wraps the ring over many tiles, so the stage index
and the barrier parity carry across tile boundaries.  Each case is checked against an fp64 product and for run-to-run
identical bits.  (The 32-wide ring of the split-bf16 convolutions has no stand-alone entry point; the forward tests of
test_gpu_parity.py run it at BLOCK_N 64 and 128, 1..9 taps and 128..1024 channels per tap.)"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

M_WRAP = 128 * 132 * 3 + 100   # ~3 tiles per CTA per 128-column slab on 132 SMs, ragged last tile
N = 256


def _split_bf16(t):
    hi = t.bfloat16()
    lo = (t - hi.float()).bfloat16()
    return torch.cat([hi, lo], dim=1).contiguous()


@pytest.mark.parametrize("epi", [0, 1, 2])
@pytest.mark.parametrize("K", [64, 192, 320])
@pytest.mark.parametrize("bn", [64, 128])
def test_gemm_x3_ring_wraps(dev, lib, bn, K, epi):
    from gdrnpp_bop2022_b200 import _lib as L

    M = M_WRAP
    g = torch.Generator().manual_seed(1000 * bn + 10 * K + epi)
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
