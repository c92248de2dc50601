"""Store what the REFERENCE's own code computes as test fixtures under tests/golden/, so that the comparisons against it
run from a plain checkout (the reference project is not needed by the tests).

  GDRN_REFERENCE_SRC=<reference checkout> python -c "import __graft_entry__ as g; g.build()"   # -> oracle/_ref/
  python tools/make_golden_ref.py --cpu  [--out tests/golden]   # libfps_ref.so, libupnp_ceres_ref.so (no GPU needed)
  python tools/make_golden_ref.py --cuda [--out tests/golden]   # ransac_voting / torch_nndistance_aten / flow_cuda

--cpu writes ref_cpu_golden.npz (FPS indices, uncertainty-PnP minimisers).  --cuda writes ref_cuda_golden.json: SHA-256
digests (first 64 bits) of the raw bytes of every output of the reference CUDA extensions on the seeded inputs of
tests/test_gpu_parity.py (the tests compare ours bit for bit, so a digest is the whole comparison).
"""
import argparse
import ctypes
import hashlib
import importlib.util
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REFDIR = os.path.join(ROOT, "oracle", "_ref")

FPS_CASES = ((1, 1), (7, 7), (100, 16), (3000, 64), (20000, 128))


def digest(t):
    """First 64 bits of the SHA-256 of the raw bytes of a tensor / array (bool as uint8)."""
    import torch

    if torch.is_tensor(t):
        t = t.detach().cpu()
        if t.dtype == torch.bool:
            t = t.to(torch.uint8)
        t = t.contiguous().numpy()
    return hashlib.sha256(np.ascontiguousarray(t).tobytes()).hexdigest()[:16]


def make_cpu(out_dir):
    from test_oracle_pinning import _upnp_problem

    fps = ctypes.CDLL(os.path.join(REFDIR, "libfps_ref.so"))
    ceres = ctypes.CDLL(os.path.join(REFDIR, "libupnp_ceres_ref.so"))
    g = {}
    rs = np.random.RandomState(5)   # the point sets of test_oracle_pinning.py::test_fps_oracle_matches_reference_build
    for pn, sn in FPS_CASES:
        pts = (rs.rand(pn, 3).astype(np.float32) - 0.5) * 0.3
        if pn == 100:
            pts[10:20] = pts[0]  # duplicates -> zero distances / ties
        idx = np.zeros(sn, np.int32)
        fps.farthest_point_sampling_init_center(pts.ctypes.data_as(ctypes.c_void_p), idx.ctypes.data_as(ctypes.c_void_p),
                                                len(pts), sn)
        g["fps_%d_%d" % (len(pts), sn)] = idx
    pts = np.random.RandomState(0).uniform(-0.1, 0.1, (8192, 3)).astype(np.float32)   # test_oracle_pinning.py's 8192-point set
    idx = np.zeros(64, np.int32)
    fps.farthest_point_sampling_init_center(pts.ctypes.data_as(ctypes.c_void_p), idx.ctypes.data_as(ctypes.c_void_p), 8192, 64)
    g["fps_8192_64"] = idx

    def solve(p2, p3, w, K, init):
        res = np.zeros(6)
        a2, a3, aw, aK, ai = (np.ascontiguousarray(x, np.float64) for x in (p2, p3, w, K, init))
        ceres.upnp_ceres_ref(*(a.ctypes.data_as(ctypes.c_void_p) for a in (a2, a3, aw, aK, ai)),
                             res.ctypes.data_as(ctypes.c_void_p), int(p2.shape[0]), None)
        return res

    # tests/test_oracle_pinning.py::test_upnp_oracle_pinned_to_vendored_ceres
    rs = np.random.RandomState(3)
    sols = []
    for trial in range(12):
        K, rt, p2, p3, w, init = _upnp_problem(rs, 8 + trial, 0.0 if trial % 2 == 0 else 0.5)
        sols.append(solve(p2, p3, w, K, init))
    g["upnp_pinning"] = np.array(sols)
    # tests/test_gpu_parity.py::test_upnp_vs_vendored_ceres_and_epnp_wrapper
    rs = np.random.RandomState(21)
    probs = [_upnp_problem(rs, 9, 0.0 if i % 2 == 0 else 0.4) for i in range(10)]
    g["upnp_device"] = np.array([solve(p2, p3, w, K, init) for (K, _, p2, p3, w, init) in probs])
    path = os.path.join(out_dir, "ref_cpu_golden.npz")
    np.savez_compressed(path, **g)
    print(path)


def load_ext(name):
    import torch  # noqa: F401  (libtorch must be loaded first)

    path = os.path.join(REFDIR, name, name + ".so")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_cuda(out_dir):
    import torch
    from test_gpu_parity import NND_REF_SHAPE, VOTING_REF_CASES, _flow_inputs, _voting_inputs, nnd_ref_inputs

    dev = torch.device("cuda:0")
    g = {"device": torch.cuda.get_device_name(0)}
    rv = load_ext("ransac_voting")
    for tn, vn, hn, seed in VOTING_REF_CASES:
        direct, coords, idxs = _voting_inputs(tn, vn, hn, seed)
        D, C, I = (torch.from_numpy(a).to(dev) for a in (direct, coords, idxs))
        for vp in (False, True):
            gen = rv.generate_hypothesis_vanishing_point if vp else rv.generate_hypothesis
            vote = rv.voting_for_hypothesis_vanishing_point if vp else rv.voting_for_hypothesis
            hyp = gen(D, C, I)
            inl = torch.zeros((hn, vn, tn), dtype=torch.uint8, device=dev)
            vote(D, C, hyp, inl, 0.99 if vp else 0.999)
            torch.cuda.synchronize()
            key = "voting_%d_%d_%d_%d_vp%d" % (tn, vn, hn, seed, int(vp))
            g[key + "_hyp"] = digest(hyp)
            g[key + "_inliers"] = digest(inl)
    nd = load_ext("torch_nndistance_aten")
    b, n, m = NND_REF_SHAPE
    a, bb = (torch.from_numpy(x).to(dev) for x in nnd_ref_inputs())
    d1 = torch.zeros(b, n, device=dev); d2 = torch.zeros(b, m, device=dev)
    i1 = torch.zeros(b, n, dtype=torch.int32, device=dev); i2 = torch.zeros(b, m, dtype=torch.int32, device=dev)
    assert nd.nnd_forward_cuda(a, bb, d1, d2, i1, i2) == 1
    torch.cuda.synchronize()
    g["nnd"] = [digest(x) for x in (d1, d2, i1, i2)]
    fl = load_ext("flow_cuda")
    for B, H, W in ((1, 8, 8), (2, 120, 160), (8, 480, 640)):
        ds, dt, KT, Kinv = _flow_inputs(B, H, W, seed=H)
        f, v = fl.forward(*(torch.from_numpy(x).to(dev) for x in (ds, dt, KT, Kinv)))
        torch.cuda.synchronize()
        g["flow_%d_%d_%d" % (B, H, W)] = [digest(f), digest(v)]
    path = os.path.join(out_dir, "ref_cuda_golden.json")
    with open(path, "w") as fh:
        json.dump(g, fh, indent=1, sort_keys=True)
    print(path)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--cuda", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.cpu:
        make_cpu(args.out)
    if args.cuda:
        make_cuda(args.out)
