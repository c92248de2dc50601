"""Micro-benchmarks of the native ops BASELINE.json's north_star names (FPS, RANSAC voting, chamfer, flow, depth
rasteriser, fast depth refine, uncertainty-PnP) at the SURVEY.md §8(d) shapes, plus BASELINE configs[2] / configs[4].

Used by bench.py (`native_ops` record of the default line, or `--workload <op>` for a single op).  Every record:
achieved HBM GB/s (or FP32 GFLOP/s for chamfer) from the ALGORITHMIC bytes/flops of SURVEY.md §8(d) over the
CUDA-event time, against MEASURED_PEAKS.json; the reference's own CUDA build (oracle/_ref/<mod>.so, built unmodified for
sm_90a) timed beside ours for voting / nnd / flow; the reference's CPU path for FPS (its .cpp, single thread) and the
CPU port for uncertainty-PnP, with the core count.  The oracle / _ref modules are baselines here, never the thing measured.

Timing: CUDA events around every call on the launching stream; a 256 MB memset evicts the 50 MB L2 before each timed
call ("l2": "flushed"); 3 warm-up calls.
"""
import ctypes
import importlib.util
import os
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
# oracle/build_ref.py builds the reference arm only when GDRN_REFERENCE_SRC names a reference checkout at build() time
REF_NOT_BUILT = "not built (oracle/_ref absent: set GDRN_REFERENCE_SRC for build())"


def _load_ref_ext(name):
    path = os.path.join(ROOT, "oracle", "_ref", name, name + ".so")
    if not os.path.exists(path):
        return None
    try:
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    except Exception:  # noqa: BLE001
        return None


class _Timer:
    def __init__(self, dev):
        self.dev = dev
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def time(self, fn, iters=10, warmup=3):
        """mean ms of fn() over `iters` calls, each preceded by an L2 flush (not timed)."""
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        tot = 0.0
        for _ in range(iters):
            self.flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            tot += e0.elapsed_time(e1)
        return tot / iters


def _rec(op, shape, ms, alg_bytes=None, alg_flops=None, peaks=None, **extra):
    r = {"op": op, "shape": shape, "ms": ms, "l2": "flushed (256 MB memset) before every timed call"}
    if alg_bytes is not None:
        gbs = alg_bytes / (ms * 1e-3) / 1e9
        r.update({"algorithmic_bytes": int(alg_bytes), "achieved": gbs, "unit": "GB/s", "bound": "hbm",
                  "peak": peaks["hbm_gbs"], "frac": gbs / peaks["hbm_gbs"]})
    if alg_flops is not None:
        gf = alg_flops / (ms * 1e-3) / 1e9
        r.update({"algorithmic_flops": int(alg_flops), "achieved": gf, "unit": "GFLOP/s", "bound": "fp32-alu",
                  "peak": peaks["fp32_gflops"], "frac": gf / peaks["fp32_gflops"]})
    r.update(extra)
    return r


# ------------------------------------------------------------------------------------------------------------- ops
def bench_fps(dev, T, peaks):
    from gdrnpp_bop2022_b200 import native_ops

    out = []
    refso = os.path.join(ROOT, "oracle", "_ref", "libfps_ref.so")
    ref = ctypes.CDLL(refso) if os.path.exists(refso) else None
    for name, b, pn, sn in (("fps 64 clouds pn=8192 sn=64", 64, 8192, 64), ("fps mesh pn=50000 sn=256", 8, 50000, 256)):
        pts = ((torch.rand(b, pn, 3, generator=torch.Generator().manual_seed(pn)) - 0.5) * 0.2).to(dev)
        ms = T.time(lambda: native_ops.farthest_point_sampling_idx(pts, sn))
        extra = {"clouds_per_s": b / (ms * 1e-3), "note": "latency bound: sn dependent arg-max steps per cloud, one CTA per cloud"}
        if ref is not None:   # the reference's own .cpp (single thread despite -fopenmp: it has no pragmas)
            p = np.ascontiguousarray(pts[0].cpu().numpy())
            idx = np.zeros(sn, np.int32)
            t0 = time.perf_counter()
            ref.farthest_point_sampling_init_center(p.ctypes.data_as(ctypes.c_void_p), idx.ctypes.data_as(ctypes.c_void_p), pn, sn)
            extra["cpu_reference_ms_per_cloud"] = (time.perf_counter() - t0) * 1e3
            extra["cpu_cores"] = 1
            extra["cpu_kind"] = "reference (farthest_point_sampling.cpp compiled into oracle/_ref/libfps_ref.so)"
        else:
            extra["cpu_kind"] = REF_NOT_BUILT
        out.append(_rec(name, {"batch": b, "pn": pn, "sn": sn}, ms, alg_bytes=b * (12 * pn + 4 * sn), peaks=peaks, **extra))
    return out


def bench_voting(dev, T, peaks):
    from gdrnpp_bop2022_b200.native_ops import ransac_voting as rv

    tn, vn, hn = 30000, 9, 128
    rs = np.random.RandomState(0)
    coords = torch.from_numpy((rs.rand(tn, 2) * 640).astype(np.float32)).to(dev)
    d = rs.randn(tn, vn, 2).astype(np.float32)
    direct = torch.from_numpy(d / np.linalg.norm(d, axis=2, keepdims=True)).to(dev)
    idxs = torch.from_numpy(rs.randint(0, tn, (hn, vn, 2)).astype(np.int32)).to(dev)
    hyp = rv.generate_hypothesis(direct, coords, idxs)
    inl = torch.zeros((hn, vn, tn), dtype=torch.uint8, device=dev)
    rd = 8 * tn * vn + 8 * tn + 8 * hn * vn
    ms_mask = T.time(lambda: rv.voting_for_hypothesis(direct, coords, hyp, inl, 0.999))
    ms_cnt = T.time(lambda: rv.vote_count(direct, coords, hyp, 0.999))
    ms_gen = T.time(lambda: rv.generate_hypothesis(direct, coords, idxs))
    shape = {"tn": tn, "vn": vn, "hn": hn}
    recs = [_rec("voting_for_hypothesis (u8 inlier mask, reference contract)", shape, ms_mask, alg_bytes=rd + hn * vn * tn, peaks=peaks),
            _rec("rv_vote_count (fused vote + count, no mask)", shape, ms_cnt, alg_bytes=rd + 4 * hn * vn, peaks=peaks,
                 note="compute (FP32 ALU) bound once the mask write is gone: hn*vn*tn = 34.6 M angle tests"),
            _rec("generate_hypothesis", shape, ms_gen, alg_bytes=8 * hn * vn * 2 * 2 + 8 * hn * vn + 8 * hn * vn, peaks=peaks,
                 note="launch-latency bound (1152 hypotheses)")]
    ref = _load_ref_ext("ransac_voting")
    if ref is not None:
        rinl = torch.zeros_like(inl)
        recs[0]["reference_cuda_ms"] = T.time(lambda: ref.voting_for_hypothesis(direct, coords, hyp, rinl, 0.999))
        recs[0]["reference_cuda_kind"] = "reference ransac_voting_kernel.cu built unmodified for sm_90a (oracle/_ref)"
        # the reference round = mask vote + torch.sum over tn (ransac_voting_gpu.py:56-60)
        recs[1]["reference_cuda_ms"] = T.time(lambda: (ref.voting_for_hypothesis(direct, coords, hyp, rinl, 0.999), torch.sum(rinl, 2)))
        recs[1]["reference_cuda_kind"] = "reference vote kernel + torch.sum(inlier, 2), what one reference RANSAC round costs"
        recs[2]["reference_cuda_ms"] = T.time(lambda: ref.generate_hypothesis(direct, coords, idxs))
    else:
        for r in recs[:3]:
            r["reference_cuda_kind"] = REF_NOT_BUILT
    return recs


def bench_nnd(dev, T, peaks):
    from gdrnpp_bop2022_b200.native_ops import torch_nndistance_aten as mine

    b, n, m = 64, 2048, 2048
    g = torch.Generator().manual_seed(0)
    a, bb = torch.rand(b, n, 3, generator=g).to(dev), torch.rand(b, m, 3, generator=g).to(dev)
    d1, d2 = torch.zeros(b, n, device=dev), torch.zeros(b, m, device=dev)
    i1, i2 = torch.zeros(b, n, dtype=torch.int32, device=dev), torch.zeros(b, m, dtype=torch.int32, device=dev)
    ms = T.time(lambda: mine.nnd_forward_cuda(a, bb, d1, d2, i1, i2))
    rec = _rec("nnd_forward_cuda (chamfer, both directions)", {"b": b, "n": n, "m": m}, ms, alg_flops=16.0 * n * m * b, peaks=peaks,
               hbm_bytes=b * (12 * (n + m) + 8 * (n + m)))
    ref = _load_ref_ext("torch_nndistance_aten")
    if ref is not None:
        rec["reference_cuda_ms"] = T.time(lambda: ref.nnd_forward_cuda(a, bb, d1, d2, i1, i2))
        rec["reference_cuda_kind"] = "reference nnd_cuda_kernel.cu built unmodified for sm_90a (oracle/_ref)"
    else:
        rec["reference_cuda_kind"] = REF_NOT_BUILT
    return [rec]


def bench_flow(dev, T, peaks):
    from gdrnpp_bop2022_b200.native_ops import flow_cuda

    B, H, W = 8, 480, 640
    g = torch.Generator().manual_seed(0)
    ds = (torch.rand(B, 1, H, W, generator=g) * 0.2 + 0.6).to(dev)
    dt = (torch.rand(B, 1, H, W, generator=g) * 0.2 + 0.6).to(dev)
    K = torch.tensor([[572.4, 0, 320.0], [0, 573.6, 240.0], [0, 0, 1]], dtype=torch.float32)
    T34 = torch.eye(4)[:3][None].repeat(B, 1, 1)
    T34[:, :, 3] = torch.randn(B, 3, generator=g) * 0.001
    KT = (K[None] @ T34).contiguous().to(dev)
    Kinv = torch.linalg.inv(K)[None].repeat(B, 1, 1).contiguous().to(dev)
    ms = T.time(lambda: flow_cuda.forward(ds, dt, KT, Kinv))
    rec = _rec("flow_cuda.forward", {"B": B, "H": H, "W": W}, ms, alg_bytes=20 * B * H * W, peaks=peaks,
               note="includes the torch.empty of the two outputs, like the reference's at::zeros")
    ref = _load_ref_ext("flow_cuda")
    if ref is not None:
        rec["reference_cuda_ms"] = T.time(lambda: ref.forward(ds, dt, KT, Kinv))
        rec["reference_cuda_kind"] = "reference flow_cuda_kernel.cu built unmodified for sm_90a (oracle/_ref)"
    else:
        rec["reference_cuda_kind"] = REF_NOT_BUILT
    return [rec]


def _mesh_and_rois(dev, n=64, subdiv=5):
    from gdrnpp_bop2022_b200.renderer import Model3D
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    v, f = make_icosphere_mesh(subdiv, (0.12, 0.09, 0.1))   # subdiv 5: 10242 vertices, 20480 faces
    rs = np.random.RandomState(1)
    poses, Ks = [], []
    for _ in range(n):
        ax = rs.randn(3)
        ax /= np.linalg.norm(ax)
        ang = rs.rand() * 3
        Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        R = np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * Kx @ Kx
        t = np.array([rs.randn() * 0.02, rs.randn() * 0.02, 0.5 + rs.rand() * 0.3])
        poses.append(np.hstack([R, t[:, None]]))
        Ks.append(np.array([[110.0 + 10 * rs.rand(), 0, 32 + rs.randn()], [0, 112.0, 31 + rs.randn()], [0, 0, 1]]))
    return (Model3D(v, f, device=dev), torch.from_numpy(np.stack(poses).astype(np.float32)).to(dev),
            torch.from_numpy(np.stack(Ks).astype(np.float32)).to(dev))


def bench_raster(dev, T, peaks):
    from gdrnpp_bop2022_b200.renderer import depth_refine, render_depth

    n, hw = 64, 64
    model, poses, Ks = _mesh_and_rois(dev, n)
    ms = T.time(lambda: render_depth(model, poses, Ks, hw, hw))
    nv, nf = model.vertices.shape[0], model.faces.shape[0]
    recs = [_rec("rast_render_meshes (64 ROI renders of one mesh)", {"rois": n, "V": nv, "F": nf, "H": hw, "W": hw}, ms,
                 alg_bytes=n * (12 * nv + 12 * nf + 4 * hw * hw), peaks=peaks, renders_per_s=n / (ms * 1e-3),
                 note="mesh is L2-resident after the first ROI; bound by triangle set-up + 64-bit atomicMin, not HBM",
                 reference_note="reference vispy renderer: 7.96 ms per 640x480 render incl. readback "
                                "(lib/render_vispy/renderer.py:564, hardware not stated); no GL on this box")]
    # fast depth refine, 2 iterations (render + refine step each), configs[2]'s refinement half
    sensor = render_depth(model, poses, Ks, hw, hw) * 1.02
    xyz = torch.rand(n, 3, hw, hw, device=dev) - 0.5
    mask = torch.rand(n, 1, hw, hw, device=dev)
    rot, trans = poses[:, :, :3].contiguous(), poses[:, :, 3].contiguous()
    ms2 = T.time(lambda: depth_refine(model, rot, trans, Ks, xyz, mask, sensor, iters=2, thresh=0.8))
    recs.append(_rec("depth_refine (2 x [render + weighted-median step])", {"rois": n, "F": nf, "iters": 2}, ms2,
                     alg_bytes=2 * n * (12 * nv + 12 * nf + 4 * hw * hw + 28 * hw * hw), peaks=peaks, rois_per_s=n / (ms2 * 1e-3),
                     reference_note="reference: 2 GL draws + 4 glReadPixels per ROI on one CPU thread "
                                    "(engine/gdrn_evaluator.py:515-561)"))
    return recs


def bench_upnp(dev, T, peaks, cpu=True):
    from gdrnpp_bop2022_b200 import native_ops

    n, pn = 512, 9
    rs = np.random.RandomState(3)
    K = np.array([[400.0, 0, 128], [0, 400, 128], [0, 0, 1]])
    P2, P3, Wt, init = [], [], [], []
    for _ in range(n):
        rt = rs.rand(6)
        p3 = rs.rand(pn, 3)
        th = np.linalg.norm(rt[:3])
        k = rt[:3] / th
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
        q = p3 @ R.T + rt[3:]
        p2 = np.stack([K[0, 0] * q[:, 0] / q[:, 2] + K[0, 2], K[1, 1] * q[:, 1] / q[:, 2] + K[1, 2]], 1) + rs.randn(pn, 2) * 0.3
        P2.append(p2); P3.append(p3); init.append(rt + rs.rand(6) * 0.1)
        Wt.append(np.stack([1 + rs.rand(pn), 0.1 * rs.randn(pn), 1 + rs.rand(pn)], 1))
    t = lambda a: torch.from_numpy(np.stack(a)).to(dev)
    a2, a3, aw, ai = t(P2), t(P3), t(Wt), t(init)
    Kd = torch.from_numpy(np.tile(K[None], (n, 1, 1))).to(dev)
    ms = T.time(lambda: native_ops.uncertainty_pnp_batched(a2, a3, aw, Kd, ai))
    rec = _rec("upnp_batched (LM, fp64, one warp per problem)", {"problems": n, "pn": pn}, ms, alg_bytes=n * 64 * pn, peaks=peaks,
               problems_per_s=n / (ms * 1e-3), note="latency bound (fp64 LM iterations), not HBM")
    if cpu:
        from oracle import ops_oracle as OO   # CPU port (libceres is absent: the reference's own build cannot run)

        k = 8
        t0 = time.perf_counter()
        for i in range(k):
            OO.uncertainty_pnp(P2[i], P3[i], Wt[i], K, init[i])
        rec["cpu_port_ms_per_problem"] = (time.perf_counter() - t0) * 1e3 / k
        rec["cpu_cores"] = 1
        rec["cpu_kind"] = "port (numpy LM restatement of uncertainty_pnp.cpp; Ceres itself is not available)"
    return [rec]


def bench_config2(dev, T, peaks, precision="bf16x3"):
    """BASELINE configs[2]: batch = 64 ROIs + fast depth refine (CUDA rasteriser, 2 iterations) + chamfer b=64."""
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg
    from gdrnpp_bop2022_b200.native_ops import torch_nndistance_aten as nndm
    from gdrnpp_bop2022_b200.renderer import depth_refine, get_K_crop_resize, render_depth
    from gdrnpp_bop2022_b200.synthetic import make_batch, make_state_dict

    B = 64
    model = GDRN_DoubleMask(default_cfg(with_maps=True), max_batch=B, precision=precision)
    model.load_state_dict(make_state_dict())
    model.to(dev)
    b = {k: v.to(dev) for k, v in make_batch(B=B, seed=3).items()}
    mesh, _, _ = _mesh_and_rois(dev, 1)
    kw = dict(roi_classes=b["roi_classes"], roi_coord_2d=b["roi_coord_2d"], roi_cams=b["roi_cams"], roi_centers=b["roi_centers"],
              roi_whs=b["roi_whs"], roi_extents=b["roi_extents"], resize_ratios=b["resize_ratios"])
    scale = 64.0 / b["resize_ratios"]
    K_crop = get_K_crop_resize(b["roi_cams"], b["roi_centers"] - scale.view(B, 1) / 2, b["resize_ratios"].view(B, 1))
    out0 = model(b["roi_img"], **kw)
    poses0 = torch.cat([out0["rot"], (out0["trans"] * 1.03)[:, :, None]], dim=2).contiguous()
    sensor = render_depth(mesh, poses0, K_crop, 64, 64)     # "sensor" = the object a little farther along the ray
    n_pts = 2048
    model_pts = mesh.vertices[torch.randperm(mesh.vertices.shape[0], device=dev)[:n_pts]].contiguous()
    d1, d2 = torch.zeros(B, n_pts, device=dev), torch.zeros(B, n_pts, device=dev)
    i1, i2 = torch.zeros(B, n_pts, dtype=torch.int32, device=dev), torch.zeros(B, n_pts, dtype=torch.int32, device=dev)

    def step():
        out = model(b["roi_img"], **kw)
        xyz = torch.cat([out["coor_x"], out["coor_y"], out["coor_z"]], dim=1)
        t2 = depth_refine(mesh, out["rot"], out["trans"], K_crop, xyz, out["mask"], sensor, iters=2, thresh=0.8)
        # chamfer between the model points under the refined pose and under the initial pose (b=64, n=m=2048)
        pa = (model_pts[None] @ out["rot"].transpose(1, 2) + t2[:, None]).contiguous()
        pb = (model_pts[None] @ out["rot"].transpose(1, 2) + out["trans"][:, None]).contiguous()
        nndm.nnd_forward_cuda(pa, pb, d1, d2, i1, i2)
        return t2

    ms = T.time(step, iters=8)
    return [{"op": "configs[2]: forward(+maps) + depth refine x2 + chamfer", "shape": {"B": B, "F": int(mesh.faces.shape[0]), "chamfer_n": n_pts},
             "precision": precision, "ms": ms, "rois_per_s": B / (ms * 1e-3), "l2": "flushed before every timed step"}]


def bench_config4(dev, T, peaks, precision="bf16x3"):
    """BASELINE configs[4] on one GPU: the YCB-V 21-object test_gdrn pose path per image -- 5 synthetic detections per
    640x480 image -> GdrnPredictor.preprocessing (GPU crops) -> inference (B = 5) -> postprocessing (host dict), the
    batching test_gdrn.sh effectively runs (SURVEY.md 3.1)."""
    from gdrnpp_bop2022_b200.predictor import GdrnPredictor
    from gdrnpp_bop2022_b200.synthetic import YCBV_K, make_state_dict

    rs = np.random.RandomState(5)
    objs = {i + 1: "obj_%06d" % (i + 1) for i in range(21)}
    extents = {i + 1: (rs.rand(3) * 0.2 + 0.05).astype(np.float32) for i in range(21)}
    pred = GdrnPredictor(cam=np.array(YCBV_K, np.float32), objs=objs, extents=extents, state_dict=make_state_dict(), device=dev,
                         precision=precision, use_pnp=False)   # test_gdrn's cfg: TEST.USE_PNP=False (YCB-V config)
    image = rs.randint(0, 256, (480, 640, 3)).astype(np.uint8)

    def dets():
        cx, cy = rs.rand(5) * 440 + 100, rs.rand(5) * 280 + 100
        bw, bh = rs.rand(5) * 160 + 40, rs.rand(5) * 160 + 40
        return np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2, np.full(5, 0.9), np.full(5, 0.9), rs.randint(0, 21, 5)], 1).astype(np.float32)

    D = [dets() for _ in range(8)]
    state = {"i": 0}

    def step():
        d = D[state["i"] % 8]
        state["i"] += 1
        data = pred.preprocessing(d, image)
        out = pred.inference(data)
        return pred.postprocessing(data, out)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    n = 30
    t0 = time.perf_counter()   # timed like engine/gdrn_evaluator.py:707-751 (perf_counter + synchronize inside inference)
    for _ in range(n):
        step()
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / n
    return [{"op": "configs[4]: per-image pose path, 5 ROIs per image (preprocessing + inference + postprocessing)",
             "shape": {"rois_per_image": 5, "image": "480x640"}, "precision": precision, "ms": dt * 1e3,
             "images_per_s": 1.0 / dt, "rois_per_s": 5.0 / dt,
             "note": "static per-batch-size input buffers + one CUDA graph per batch size (GdrnPredictor.use_cuda_graph); timed like gdrn_evaluator.py:707-751"}]


WORKLOADS = {"fps": bench_fps, "voting": bench_voting, "nnd": bench_nnd, "flow": bench_flow, "raster": bench_raster,
             "upnp": bench_upnp, "refine": bench_config2, "ycbv5": bench_config4}


def peaks_with_fp32(peaks):
    p = dict(peaks)
    mhz = p.get("sm_max_mhz") or 1980.0
    p["fp32_gflops"] = 132 * 128 * 2 * mhz * 1e6 / 1e9   # H100 SXM: 132 SMs x 128 FMA lanes x 2 FLOP x clock
    return p


def run(dev, peaks, which=None, precision="bf16x3"):
    T = _Timer(dev)
    peaks = peaks_with_fp32(peaks)
    out = []
    for name, fn in WORKLOADS.items():
        if which and name not in which:
            continue
        try:
            if name in ("refine", "ycbv5"):
                out += fn(dev, T, peaks, precision)
            else:
                out += fn(dev, T, peaks)
        except Exception as e:  # noqa: BLE001  (a failing micro-benchmark must not take the headline down)
            out.append({"op": name, "error": "%s: %s" % (type(e).__name__, e)})
    return out
