"""Generate tests/golden/gemm_x3_digests.json: SHA-256 digests of gdrn_gemm_x3 outputs (split-bf16 GEMM, parity mode) from
seeded inputs, at the six ConvNeXt stage-1..3 MLP shapes of bench_gemm_x3.py (B = 64, the tile widths an H100's 132 SMs
give them), a downsample shape and the small-batch (B = 5) shapes that run 64-wide tiles.  Every output element comes from
a fixed wgmma sequence and a fixed epilogue, so a change to the kernel's plumbing must reproduce these bytes exactly.

  python tools/make_golden_gemm_x3.py [--out PATH]     needs a GPU

tests/test_gemm_x3_reg_epilogue.py recomputes the digests with `digest_case` and compares."""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden", "gemm_x3_digests.json")

# (name, M, N, K, epi, block_n); epi 0 = store fp32 (+bias), 1 = GELU -> [hi | lo] bf16, 2 = in-place x += gamma * (.)
CASES = [
    ("stage-1 fc1", 65536, 1024, 256, 1, 256), ("stage-1 fc2", 65536, 256, 1024, 2, 256),
    ("stage-2 fc1", 16384, 2048, 512, 1, 256), ("stage-2 fc2", 16384, 512, 2048, 2, 256),
    ("stage-3 fc1", 4096, 4096, 1024, 1, 256), ("stage-3 fc2", 4096, 1024, 4096, 2, 256),
    ("stage-2 downsample", 16384, 512, 1024, 0, 256),
    ("B=5 stage-3 fc2", 320, 1024, 4096, 2, 64),
    ("B=5 stage-3 fc1 at 64", 320, 4096, 1024, 1, 64),
    ("B=5 stage-3 downsample", 320, 1024, 2048, 0, 64),
]


def _split_bf16(t):
    import torch

    hi = t.bfloat16()
    lo = (t - hi.float()).bfloat16()
    return torch.cat([hi, lo], dim=1).contiguous()


def digest_case(lib, dev, case):
    """Run one case from its seeded inputs and return the SHA-256 hex digest of the whole output buffer."""
    import numpy as np
    import torch

    from gdrnpp_bop2022_b200 import _lib as L

    name, M, N, K, epi, bn = case
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K + epi)
    A = _split_bf16(torch.randn(M, K, generator=g)).to(dev)
    W = _split_bf16(torch.randn(N, K, generator=g) / np.sqrt(K)).to(dev)
    bias, gamma = torch.randn(N, generator=g).to(dev), torch.rand(N, generator=g).to(dev)
    if epi == 1:
        out = torch.zeros((M, 2 * N), dtype=torch.bfloat16, device=dev)
    else:
        out = torch.randn(M, N, generator=g).to(dev) if epi == 2 else torch.zeros((M, N), dtype=torch.float32, device=dev)
    L.check(lib.gdrn_gemm_x3(L.ptr(A), L.ptr(W), L.ptr(bias), L.ptr(gamma), L.ptr(out), L.ptr(out), M, N, K, epi, bn,
                             L.current_stream()), "gemm_x3 " + name)
    torch.cuda.synchronize()
    return hashlib.sha256(out.view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=GOLDEN)
    args = ap.parse_args()
    import torch

    from gdrnpp_bop2022_b200 import _lib as L

    dev = torch.device("cuda:0")
    lib = L.lib()
    rec = {"device": torch.cuda.get_device_name(dev), "cases": []}
    for case in CASES:
        rec["cases"].append({"name": case[0], "M": case[1], "N": case[2], "K": case[3], "epi": case[4], "block_n": case[5],
                             "sha256": digest_case(lib, dev, case)})
        print(json.dumps(rec["cases"][-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", args.out)


if __name__ == "__main__":
    main()
