"""Fast depth refine (csrc/raster.cu depth_refine_kernel) one stage at a time against the f64 oracle
(oracle/depth_refine_oracle.py).

Every stage is checked on the kernel's own inputs to it, read from gdrn_depth_refine_trace: the mask normalisation and
the weights, their sum, max and min, the cut and the selection, the median, the centroid, the ray and t.  An error
upstream therefore can neither hide nor leak into a later check.

Max, min, count, the selection outside a relative band of 2^-21 around the cut, and the median are exact.  The other
bars are derived from the f32 arithmetic (stated next to each) and are at most 4x the largest error measured on an H100
(80GB HBM3, 700 W power limit); the measured maxima are listed next to the bars in BARS.  The driver tests then check
renderer.depth_refine step by step against the f64 step fed with the library's own renders, and against f64 renders
(oracle/raster_oracle.py).

The oracle and sensor-crop tests at the top need no GPU.
"""
import math

import numpy as np
import pytest
import torch

from oracle import depth_refine_oracle as DO
from oracle import ops_oracle as OO

ULP = 2.0 ** -24   # unit roundoff of f32

# quantity -> (bar, largest value measured on the H100 above)
BARS = {
    # |w - w64| in units of ULP * |q| * |m64| (q = ||xyz||, or sum_j |R_2j x_j| for coor-z): the f32 norm or dot
    # product, the product with the mask and the mask itself (the min-max subtract and divide, or expf's 2 ulp and the
    # sigmoid's divide); derived <= 4, 6, 8 for mask modes 0, 1, 2
    "w_mask0": (4.0, 2.68),
    "w_mask1": (6.0, 4.41),
    "w_mask2": (8.0, 4.3),
    # |sum - fsum(w)| / sum|w|: the double tree sum of hw*hw f32 weights; derived <= hw^2 * 2^-53 ~ 1.8e-12, the bar is
    # 4x the measured maximum
    "sum": (6e-16, 1.85e-16),
    # |cut - cut64| / |cut64| at the f32 threshold the kernel receives: the f32 reciprocal, product and threshold
    # product; derived <= 3 ULP
    "cut": (3 * ULP, 1.51e-07),
    # |c - c64| in units of ULP * sum_i |wn_i| * (row or col): the f32 reciprocal and one f32 product per pixel;
    # derived <= 2
    "centroid": (2.0, 1.77),
    # |ray - ray64| / |ray64|: the double 3x3 inverse (a few 2^-53); the bar is 4x the measured maximum
    "ray": (8e-16, 2.22e-16),
    # |t - t64| in f32 ulps of t, t64 = t0 + ray(c) * median in f64: one rounding to f32
    "t": (0.5, 0.5),
    # driver: max |t - step64(library render)| in f32 ulps of max |t|, every stage bar above together
    "driver_t": (1.0, 0.5),
    # end to end: |t - step64(f64 render)| over the bound |ray| * max selected depth * (the render's measured relative
    # depth error) + 1 ulp of t
    "e2e_t": (0.95, 0.247),
}
MEASURED = {}


def _note(what, value, case):
    if value > MEASURED.get(what, (-1.0, None))[0]:
        MEASURED[what] = (float(value), case)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, (v, case) in sorted(MEASURED.items()):
        print(f"measured {k}: {v:.3g} at {case}")


def _ulp32(x):
    x = np.abs(np.asarray(x, np.float32))
    return np.spacing(np.maximum(x, np.float32(np.finfo(np.float32).tiny))).astype(np.float64)


def _rot(rs):
    from scipy.spatial.transform import Rotation

    ax = rs.randn(3)
    return Rotation.from_rotvec(ax / np.linalg.norm(ax) * rs.rand() * 3).as_matrix().astype(np.float32)


def make_inputs(rs, n, hw, mask_mode):
    """n ROIs of random refine inputs: xyz in [0,1), a raw mask for the mode (normalised [0,1), L1 outputs, logits),
    renders at 0.6-0.9 m with ~30 % background, sensor depth with ~10 % holes, crop intrinsics, rotations, t."""
    xyz = rs.rand(n, 3, hw, hw).astype(np.float32)
    mask = {0: rs.rand(n, hw, hw), 1: rs.randn(n, hw, hw) * 2 + 0.5, 2: rs.randn(n, hw, hw) * 4}[mask_mode].astype(np.float32)
    ren = np.where(rs.rand(n, hw, hw) < 0.7, 0.6 + 0.3 * rs.rand(n, hw, hw), 0).astype(np.float32)
    sensor = np.where(rs.rand(n, hw, hw) < 0.9, ren + 0.01 * rs.randn(n, hw, hw) + 0.02, 0).astype(np.float32)
    f = hw * (1.6 + 0.3 * rs.rand(n))
    K = np.zeros((n, 3, 3), np.float32)
    K[:, 0, 0], K[:, 1, 1], K[:, 2, 2] = f, f * (1 + 0.02 * rs.randn(n)), 1
    K[:, 0, 2], K[:, 1, 2] = hw / 2 + rs.randn(n), hw / 2 + rs.randn(n)
    R = np.stack([_rot(rs) for _ in range(n)])
    t = np.stack([rs.randn(n) * 0.05, rs.randn(n) * 0.05, 0.6 + 0.3 * rs.rand(n)], 1).astype(np.float32)
    return dict(xyz=xyz, mask=mask, ren=ren, sensor=sensor, K=K, R=R, t=t)


# ================================================================================ oracle pinning (CPU)
def test_oracle_equals_reference_restatements():
    """step equals the reference's arithmetic restated verbatim: ops_oracle.depth_refine_step (||xyz|| weights, f32
    torch norm and f32 division) and test_net_pnp.ref_coor_z_step (coor-z), on their own inputs.  The restatements
    round in f32, so t agrees to 1e-7 m."""
    from test_net_pnp import _coor_z_inputs, ref_coor_z_step

    xyz, mask, ren, sensor, K, R, t = _coor_z_inputs(3)
    n = mask.shape[0]
    mn, mx = mask.reshape(n, -1).min(1)[:, None, None], mask.reshape(n, -1).max(1)[:, None, None]
    mask_n = (mask - mn) / (mx - mn)
    for i in range(n):
        x01 = xyz[i].transpose(1, 2, 0)
        want = ref_coor_z_step(x01, mask_n[i], sensor[i], ren[i], K[i].astype(np.float64), R[i], t[i].astype(np.float64))
        got, st = DO.step(xyz[i], mask[i], ren[i], sensor[i], K[i], t[i], R=R[i], mask_mode=1, weight_mode=1)
        assert np.abs(got - want).max() < 1e-7, (i, got, want)
        want0 = OO.depth_refine_step(x01, mask_n[i], sensor[i], ren[i], K[i].astype(np.float64), t[i].astype(np.float64))
        got0, _ = DO.step(xyz[i], mask[i], ren[i], sensor[i], K[i], t[i], mask_mode=1, weight_mode=0)
        assert np.abs(got0 - want0).max() < 1e-7, (i, got0, want0)
    assert st["ns"]["sum"] == 0.0 and not st["changed"]       # ROI 3 of these inputs cancels exactly


def test_oracle_replay_equals_reference_loop():
    """replay over the numpy renderer equals the reference's two-iteration loop restated with
    ops_oracle.depth_refine_step, to the f32 rounding of that restatement."""
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    rs = np.random.RandomState(8)
    v, f = (np.asarray(a) for a in make_icosphere_mesh(2, (0.12, 0.08, 0.1)))
    R = _rot(rs)
    t0 = np.array([0.01, -0.01, 0.6])
    K = np.array([[110.0, 0, 32.3], [0, 112.0, 31.1], [0, 0, 1]], np.float32)
    pose = lambda t: np.hstack([R, np.asarray(t, np.float32)[:, None]]).astype(np.float32)
    render = lambda Rr, t: OO.render_depth(v, f, pose(t), K, 64, 64)
    sensor = render(R, t0 * 1.03).astype(np.float32)
    xyz = rs.rand(3, 64, 64).astype(np.float32)
    mask = rs.rand(64, 64).astype(np.float32)
    got, stages = DO.replay(render, xyz, mask, sensor, K, R, t0, iters=2, mask_mode=0)
    t = t0.copy()
    for _ in range(2):
        t = OO.depth_refine_step(xyz.transpose(1, 2, 0), mask, sensor, render(R, t), K.astype(np.float64), t)
    assert all(st["changed"] for st in stages) and np.abs(got - t).max() < 1e-7, (got, t)


def test_oracle_hand_worked():
    """Odd and even counts, a known centroid and ray, a negative coor-z sum, an exactly zero sum, and the empty
    selections (constant L1 mask, thresh >= 1)."""
    hw = 5
    K = np.array([[100.0, 0, 2.0], [0, 100.0, 2.0], [0, 0, 1]])
    xyz = np.zeros((3, hw, hw), np.float32)
    xyz[2] = 1.0                                    # ||xyz|| = 1: the weight is the mask
    ren = np.full((hw, hw), 0.5, np.float32)
    sensor = ren + np.arange(hw * hw, dtype=np.float32).reshape(hw, hw) * np.float32(0.001)
    t = np.array([0.0, 0.0, 0.5])
    # three equal weights at (1,1), (1,3), (3,2): count 3, median = the middle diff, centroid (5/3, 2)
    m = np.zeros((hw, hw), np.float32)
    m[1, 1] = m[1, 3] = m[3, 2] = 1.0
    got, st = DO.step(xyz, m, ren, sensor, K, t, mask_mode=0)
    assert st["ns"]["sel"].sum() == 3 and st["med"] == sensor[1, 3] - ren[1, 3]
    assert np.allclose(st["centroid"], (5 / 3, 2.0), rtol=0, atol=1e-15)
    assert np.allclose(st["ray"], [0.0, (5 / 3 - 2) / 100, 1.0], rtol=0, atol=1e-15)
    assert np.allclose(got, t + st["ray"] * st["med"], rtol=0, atol=0)
    # even count: the fourth pixel joins, the median averages the two middle diffs
    m[4, 4] = 1.0
    _, st = DO.step(xyz, m, ren, sensor, K, t, mask_mode=0)
    d = np.sort(sensor[m > 0] - ren[m > 0])
    assert st["ns"]["sel"].sum() == 4 and st["med"] == (d[1] + d[2]) / np.float32(2)
    assert st["med"] == np.median(sensor[m > 0] - ren[m > 0])
    # one pixel above the cut: count 1
    m[4, 4] = 2.0
    _, st = DO.step(xyz, m, ren, sensor, K, t, mask_mode=0)
    assert st["ns"]["sel"].sum() == 1 and st["med"] == sensor[4, 4] - ren[4, 4]
    # coor-z with R = rot(x, pi): (R xyz)_z = -z, every weight <= 0 and a negative sum; the cut comes from the most
    # negative weight, so the pixel with the largest mask is selected
    Rx = np.diag([1.0, -1.0, -1.0]).astype(np.float32)
    _, st = DO.step(xyz, m, ren, sensor, K, t, R=Rx, mask_mode=0, weight_mode=1)
    assert st["ns"]["sum"] < 0 and st["ns"]["min"] == -2.0 and st["ns"]["sel"].sum() == 1 and st["ns"]["sel"][4, 4]
    # a zero sum: no valid sensor pixel
    got, st = DO.step(xyz, m, ren, np.zeros_like(sensor), K, t, mask_mode=0)
    assert st["ns"]["sum"] == 0.0 and np.array_equal(got, t) and not st["changed"]
    # a constant L1 mask: 0 / 0, NaN cut, nothing selected, t unchanged (the reference's median would be NaN)
    got, st = DO.step(xyz, np.full((hw, hw), 0.3, np.float32), ren, sensor, K, t, mask_mode=1)
    assert np.isnan(st["ns"]["cut"]) and not st["ns"]["sel"].any() and np.array_equal(got, t)
    # thresh 1: nothing exceeds the max
    got, st = DO.step(xyz, m, ren, sensor, K, t, mask_mode=0, thresh=1.0)
    assert not st["ns"]["sel"].any() and np.array_equal(got, t) and np.isnan(DO.median([]))


def test_oracle_median_is_np_median():
    """median == np.median bit for bit on f32 arrays of odd and even length, duplicates included."""
    rs = np.random.RandomState(0)
    for n in list(range(1, 12)) + [100, 101, 4096]:
        d = (rs.randint(-50, 50, n) * 1e-3 + rs.randn(n) * 1e-6 * (rs.rand() < 0.5)).astype(np.float32)
        assert np.float32(DO.median(d)).view(np.int32) == np.median(d).view(np.int32), n


def test_oracle_mask_modes():
    """out_mask: identity, min-max and sigmoid against closed forms."""
    m = np.array([[-2.0, 0.0], [1.0, 6.0]], np.float32)
    assert np.array_equal(DO.out_mask(m, 0), m.astype(np.float64))
    assert np.array_equal(DO.out_mask(m, 1), np.array([[0.0, 0.25], [0.375, 1.0]]))
    assert np.allclose(DO.out_mask(m, 2), [[1 / (1 + math.e ** 2), 0.5], [1 / (1 + math.e ** -1), 1 / (1 + math.e ** -6)]],
                       rtol=1e-15, atol=0)


def _sensor_crops(rs, n=4):
    """Random 256x256 depth crops in metres with ~10 % holes, and the formula's 64x64 crop ((a+b)+(c+d))*0.25."""
    d = (rs.uniform(0.3, 2.5, (n, 256, 256)) * (rs.rand(n, 256, 256) > 0.1)).astype(np.float32)
    f = ((d[:, 1::4, 1::4] + d[:, 1::4, 2::4]) + (d[:, 2::4, 1::4] + d[:, 2::4, 2::4])) * np.float32(0.25)
    return d, f


def _cv2_resize(d, optimized):
    import cv2

    was = cv2.useOptimized()
    try:
        cv2.setUseOptimized(optimized)
        return np.stack([cv2.resize(x, (64, 64)) for x in d])
    finally:
        cv2.setUseOptimized(was)


def test_sensor_crop_formula_vs_cv2_resize():
    """The reference's sensor crop is cv2.resize(roi_depth, (64, 64)), bilinear 256 -> 64.  With OpenCV's optimised
    code off it equals ((a+b)+(c+d))*0.25 of the centre 2x2 of every 4x4 cell bit for bit; the default optimised path
    rounds in two passes and differs from it on a few percent of the pixels, by 1 ulp and on under 1 % by 2 ulp."""
    import cv2

    was = cv2.useOptimized()
    d, f = _sensor_crops(np.random.RandomState(0))
    assert np.array_equal(_cv2_resize(d, False).view(np.int32), f.view(np.int32))
    fast = _cv2_resize(d, True)
    assert cv2.useOptimized() == was
    diff = np.abs(fast.view(np.int32).astype(np.int64) - f.view(np.int32).astype(np.int64))
    assert diff.max() <= 2 and 0.01 < (diff > 0).mean() < 0.2 and (diff > 1).mean() < 0.01, ((diff > 0).mean(), diff.max())


# ================================================================================ GPU: the kernel against the oracle
def _T(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def run_trace(dev, inp, mask_mode, weight_mode, thresh):
    """The traced step and the production step on the same inputs; their outputs must be equal bit for bit."""
    from gdrnpp_bop2022_b200 import _lib as L
    from gdrnpp_bop2022_b200.renderer import depth_refine_trace

    g = {k: _T(dev, v) for k, v in inp.items()}
    rot = g["R"] if weight_mode == 1 else None
    tr = depth_refine_trace(g["xyz"], g["mask"], g["sensor"], g["ren"], g["K"], g["t"], rot=rot, mask_mode=mask_mode,
                            weight_mode=weight_mode, thresh=thresh)
    t = g["t"].clone()
    n, hw = inp["mask"].shape[0], inp["mask"].shape[-1]
    L.check(L.lib().gdrn_depth_refine_step(L.ptr(g["xyz"]), L.ptr(g["mask"]), mask_mode, L.ptr(g["sensor"]), L.ptr(g["ren"]),
                                           L.ptr(g["K"]), L.ptr(rot), weight_mode, L.ptr(t), n, hw, float(thresh),
                                           L.current_stream()), "gdrn_depth_refine_step")
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in tr.items()}
    assert np.array_equal(out["t"].view(np.int32), t.cpu().numpy().view(np.int32))      # trace on == trace off
    return out


def check_stages(inp, tr, mask_mode, weight_mode, thresh, case):
    """Every stage of every ROI against the oracle on the kernel's own inputs to that stage.  Returns the counts."""
    n, hw = inp["mask"].shape[0], inp["mask"].shape[-1]
    counts = []
    for i in range(n):
        xyz, raw, ren, sen = inp["xyz"][i], inp["mask"][i], inp["ren"][i], inp["sensor"][i]
        c = f"{case} roi {i}"
        # mask normalisation
        if mask_mode == 1:
            assert tr["m_lo"][i] == raw.min() and tr["m_scale"][i] == np.float32(raw.max() - raw.min()), c
        else:
            assert tr["m_lo"][i] == 0 and tr["m_scale"][i] == 1, c
        valid = (ren > 0) & (sen > 0)
        if mask_mode == 1 and tr["m_scale"][i] == 0 and valid.any():
            # a constant L1 mask (every hw = 1 ROI): 0 / 0 weights, a NaN sum and cut, nothing selected, t unchanged
            assert np.isnan(tr["w"][i][valid]).all() and np.isnan(tr["sum"][i]) and np.isnan(tr["cut"][i]), c
            assert tr["count"][i] == 0 and np.array_equal(tr["t"][i], inp["t"][i]), c
            counts.append(0)
            continue
        # weights
        m64 = DO.out_mask(raw, mask_mode)
        w64 = DO.weights(xyz, m64, ren, sen, inp["R"][i], weight_mode)
        w = tr["w"][i].astype(np.float64)
        assert (w[~valid] == 0).all(), c
        x = xyz.astype(np.float64)
        q = np.sqrt((x * x).sum(0)) if weight_mode == 0 else np.abs(inp["R"][i][2].astype(np.float64)[:, None, None] * x).sum(0)
        mag = q * np.abs(m64)
        if valid.any() and mag[valid].max() > 0:
            e = (np.abs(w - w64)[valid] / (ULP * np.maximum(mag[valid], 1e-300))).max()
            _note(f"w_mask{mask_mode}", e, c)
            assert e <= BARS[f"w_mask{mask_mode}"][0], (c, e)
        # sum, max, min
        assert tr["max"][i] == max(np.float32(0), w.max()) and tr["min"][i] == min(np.float32(0), w.min()), c
        s = math.fsum(w.ravel())
        assert tr["sum"][i] == s or abs(tr["sum"][i] - s) <= BARS["sum"][0] * np.abs(w).sum(), c
        _note("sum", abs(tr["sum"][i] - s) / max(np.abs(w).sum(), 1e-300), c)
        if s == 0.0:                                   # pose unchanged, the kernel stops before the cut
            assert tr["count"][i] == -1 and np.isnan(tr["cut"][i]), c
            assert np.array_equal(tr["t"][i], inp["t"][i]), c
            counts.append(0)
            continue
        # cut and selection, on the kernel's weights
        ns = DO.normalise_and_select(w, float(np.float32(thresh)))
        if np.isfinite(ns["cut"]) and ns["cut"] != 0:
            e = abs(np.float64(tr["cut"][i]) - ns["cut"]) / abs(ns["cut"])
            _note("cut", e, c)
            assert e <= BARS["cut"][0], (c, e)
        sel = tr["sel"][i]
        assert not (sel != ns["sel"])[~ns["amb"]].any(), (c, int((sel != ns["sel"]).sum()))
        assert tr["count"][i] == sel.sum(), c
        counts.append(int(sel.sum()))
        if not sel.any():                              # empty selection: t unchanged, nothing downstream written
            assert np.array_equal(tr["t"][i], inp["t"][i]) and np.isnan(tr["median"][i]), c
            continue
        # median of the kernel's own selection: bit-exact
        assert tr["median"][i].view(np.int32) == np.median(sen[sel] - ren[sel]).view(np.int32), c
        assert tr["median"][i] == np.float32(DO.median(sen[sel] - ren[sel])), c
        # centroid
        wn = w / tr["sum"][i]
        cy, cx = DO.centroid(wn)
        rows, cols = np.indices(w.shape, dtype=np.float64)
        for got, want, wt in ((tr["centroid"][i, 0], cy, rows), (tr["centroid"][i, 1], cx, cols)):
            scale = ULP * np.abs(wn * wt).sum()
            e = abs(got - want) / scale if scale > 0 else abs(got - want)
            _note("centroid", e, c)
            assert e <= BARS["centroid"][0], (c, got, want, e)
        # ray and t from the traced centroid and median
        r64 = DO.ray(inp["K"][i], tr["centroid"][i])
        e = np.abs(tr["ray"][i] - r64).max() / np.abs(r64).max()
        _note("ray", e, c)
        assert e <= BARS["ray"][0], (c, e)
        t64 = inp["t"][i].astype(np.float64) + r64 * np.float64(tr["median"][i])
        e = (np.abs(tr["t"][i] - t64) / _ulp32(t64)).max()
        _note("t", e, c)
        assert e <= BARS["t"][0], (c, tr["t"][i], t64, e)
        assert np.array_equal(tr["t_trace"][i], tr["t"][i]), c
    return counts


N_ROIS = {1: 300, 2: 300, 7: 200, 33: 64, 64: 33, 100: 12, 128: 8}
THRESHOLDS = (0.0, 0.5, 0.8, 0.999, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("weight_mode", [0, 1])
@pytest.mark.parametrize("mask_mode", [0, 1, 2])
@pytest.mark.parametrize("hw", sorted(N_ROIS))
def test_stages(dev, hw, mask_mode, weight_mode):
    """Every stage against the oracle for every threshold, at hw from 1 to 128 (128: the 128 KB shared-memory case;
    100 and 33: pixel counts that are not powers of two, so the sort pads with INF)."""
    rs = np.random.RandomState(hw * 10 + mask_mode * 2 + weight_mode)
    inp = make_inputs(rs, N_ROIS[hw], hw, mask_mode)
    parities = set()
    for thresh in THRESHOLDS:
        tr = run_trace(dev, inp, mask_mode, weight_mode, thresh)
        counts = check_stages(inp, tr, mask_mode, weight_mode, thresh, f"hw {hw} mask {mask_mode} w {weight_mode} thr {thresh}")
        parities |= {c % 2 for c in counts if c > 0}
        if thresh >= 1.0:
            assert max(counts) == 0
    if hw >= 7:
        assert parities == {0, 1}                   # odd and even selection counts both reached the median


def _single(hw=16):
    """One ROI whose weight is the mask (xyz = (0, 0, 1)), every render and sensor pixel valid, distinct diffs."""
    xyz = np.zeros((1, 3, hw, hw), np.float32)
    xyz[:, 2] = 1
    ren = np.full((1, hw, hw), 0.7, np.float32)
    sensor = ren + (np.arange(hw * hw, dtype=np.float32).reshape(1, hw, hw) - 100) * np.float32(1e-4)
    K = np.array([[[30.0, 0, 8.3], [0, 31.0, 7.6], [0, 0, 1]]], np.float32)
    return dict(xyz=xyz, mask=np.zeros((1, hw, hw), np.float32), ren=ren, sensor=sensor, K=K,
                R=np.eye(3, dtype=np.float32)[None], t=np.array([[0.01, -0.02, 0.7]], np.float32))


@pytest.mark.gpu
def test_edge_counts_one_two_and_ties(dev):
    """A count of 1 and of 2 (one ROI each, n = 1), and many pixels tied at the max weight with all diffs equal."""
    inp = _single()
    inp["mask"][0] = 0.5
    inp["mask"][0, 3, 4] = 1.0
    tr = run_trace(dev, inp, 0, 0, 0.8)
    check_stages(inp, tr, 0, 0, 0.8, "count 1")
    assert tr["count"][0] == 1 and tr["median"][0] == inp["sensor"][0, 3, 4] - inp["ren"][0, 3, 4]
    inp["mask"][0, 9, 2] = 1.0
    tr = run_trace(dev, inp, 0, 0, 0.8)
    check_stages(inp, tr, 0, 0, 0.8, "count 2")
    a, b = inp["sensor"][0, 3, 4] - inp["ren"][0, 3, 4], inp["sensor"][0, 9, 2] - inp["ren"][0, 9, 2]
    assert tr["count"][0] == 2 and tr["median"][0] == np.float32(0.5) * (a + b)
    # 50 pixels tied at the max, the same diff everywhere: all 50 selected at thresh 0.999, the median is that diff
    rs = np.random.RandomState(0)
    inp["mask"][0] = rs.rand(16, 16).astype(np.float32) * 0.9
    inp["mask"][0].ravel()[rs.choice(256, 50, replace=False)] = 1.0
    inp["sensor"][0] = inp["ren"][0] + np.float32(0.0123)
    tr = run_trace(dev, inp, 0, 0, 0.999)
    check_stages(inp, tr, 0, 0, 0.999, "ties")
    assert tr["count"][0] == 50 and tr["median"][0] == (inp["sensor"][0] - inp["ren"][0]).ravel()[0]


@pytest.mark.gpu
def test_edge_zero_negative_and_cancelling_sums(dev):
    """No valid sensor depth (sum 0: t unchanged); a negative coor-z sum (the cut comes from the most negative weight);
    an exactly cancelling coor-z sum (t unchanged)."""
    inp = _single()
    inp["mask"][0] = np.random.RandomState(1).rand(16, 16)
    sensor = inp["sensor"].copy()
    inp["sensor"][:] = 0
    tr = run_trace(dev, inp, 0, 0, 0.8)
    check_stages(inp, tr, 0, 0, 0.8, "no sensor")
    assert tr["sum"][0] == 0 and np.array_equal(tr["t"], inp["t"])
    inp["sensor"] = sensor
    inp["R"][0] = np.diag([1.0, -1.0, -1.0])          # (R xyz)_z = -z: every weight <= 0
    tr = run_trace(dev, inp, 0, 1, 0.8)
    check_stages(inp, tr, 0, 1, 0.8, "negative sum")
    assert tr["sum"][0] < 0 and tr["cut"][0] > 0 and tr["count"][0] > 0
    assert tr["sel"][0][np.unravel_index(np.argmax(inp["mask"][0]), (16, 16))]
    # two valid pixels whose coor-z weights are +0.5 h and -0.5 h (h = f32 sqrt(1/2)) sum to exactly 0
    h = np.float32(np.sqrt(0.5))
    inp["R"][0] = np.array([[-h, 0, -h], [0, 1, 0], [h, 0, -h]])
    inp["mask"][0] = 0
    inp["mask"][0, 2, 2] = inp["mask"][0, 5, 6] = 1
    inp["xyz"][0, :, 2, 2] = (0.5, 0.3, 0.0)
    inp["xyz"][0, :, 5, 6] = (0.0, 0.7, 0.5)
    tr = run_trace(dev, inp, 0, 1, 0.8)
    check_stages(inp, tr, 0, 1, 0.8, "cancelling sum")
    assert tr["sum"][0] == 0 and np.array_equal(tr["t"], inp["t"])


@pytest.mark.gpu
def test_edge_empty_selections(dev):
    """A constant L1 mask (0 / 0: NaN weights and cut, nothing selected) and thresh >= 1 (nothing exceeds the max)
    leave t unchanged, where the reference's np.median([]) would make it NaN."""
    inp = _single()
    inp["mask"][0] = 0.25
    tr = run_trace(dev, inp, 1, 0, 0.8)
    assert tr["m_scale"][0] == 0 and np.isnan(tr["cut"][0]) and tr["count"][0] == 0
    assert np.array_equal(tr["t"], inp["t"])
    _, st = DO.step(inp["xyz"][0], inp["mask"][0], inp["ren"][0], inp["sensor"][0], inp["K"][0], inp["t"][0], mask_mode=1)
    assert np.isnan(st["ns"]["cut"]) and not st["changed"]
    inp["mask"][0] = np.random.RandomState(2).rand(16, 16)
    for thresh in (1.0, 1.5):
        tr = run_trace(dev, inp, 0, 0, thresh)
        check_stages(inp, tr, 0, 0, thresh, f"thresh {thresh}")
        assert tr["count"][0] == 0 and np.array_equal(tr["t"], inp["t"])


@pytest.mark.gpu
def test_scale_invariance_down_to_tiny_sums(dev):
    """The refine depends on the weights only through w / sum(w), so scaling a mask_mode 0 mask by 2^k leaves t
    unchanged.  The weights here are multiples of 2^-8 in (0, 1], so w * 2^k stays exact down to k = -140 (subnormal
    weights included) and t must be bit-identical for every k.  Below sum = 2^-128 the f32 reciprocal of the sum
    overflows; the kernel then scales the weights by 2^64 and the reciprocal by 2^-64 rather than select nothing."""
    rs = np.random.RandomState(3)
    n, hw = 6, 64
    inp = make_inputs(rs, n, hw, 0)
    inp["xyz"][:] = 0
    inp["xyz"][:, 2] = rs.randint(1, 17, (n, hw, hw)) / np.float32(16)          # ||xyz|| = z exactly
    base = rs.randint(0, 17, (n, hw, hw)).astype(np.float32) / 16                # w = z * m: multiples of 2^-8
    ks = list(range(0, -141, -4)) + [-126, -127, -128, -129, -130, -131, -135, -140]
    outs, tiny = [], 0
    for k in ks:
        inp["mask"] = (base * np.float32(2.0 ** k)).astype(np.float32)
        assert np.array_equal(inp["mask"] / np.float32(2.0 ** k), base)          # the scaled mask is exact
        tr = run_trace(dev, inp, 0, 0, 0.8)
        tiny += int((np.abs(tr["sum"]) < 2.0 ** -128).sum())
        outs.append(tr)
    assert tiny > 0
    ref = outs[0]
    for k, tr in zip(ks, outs):
        assert np.array_equal(tr["count"], ref["count"]) and (ref["count"] > 0).all(), k
        assert np.array_equal(tr["sel"], ref["sel"]), k
        assert np.array_equal(tr["median"].view(np.int32), ref["median"].view(np.int32)), k
        assert np.array_equal(tr["centroid"], ref["centroid"]), k
        assert np.array_equal(tr["t"].view(np.int32), ref["t"].view(np.int32)), k
        assert not np.array_equal(tr["t"], inp["t"]), k


# ================================================================================ GPU: the driver
# the driver's f64 step recomputes the weights from the raw inputs, so its band covers the f32 weight error too (the
# largest w bar, 8 ulps) on top of the normalisation's
DRIVER_BAND = 2.0 ** -18


def _meshes(dev):
    from gdrnpp_bop2022_b200.renderer import Model3D
    from gdrnpp_bop2022_b200.synthetic import make_icosphere_mesh

    shapes = [(3, (0.12, 0.08, 0.1)), (2, (0.06, 0.09, 0.05)), (3, (0.15, 0.15, 0.07))]
    vf = [make_icosphere_mesh(s, e) for s, e in shapes]
    return [(np.asarray(v, np.float32), np.asarray(f, np.int32)) for v, f in vf], [Model3D(v, f, device=dev) for v, f in vf]


def _driver_case(dev, seed, n=12):
    from gdrnpp_bop2022_b200.renderer import render_meshes

    rs = np.random.RandomState(seed)
    vf, models = _meshes(dev)
    mesh_ids = rs.randint(0, len(models), n)
    R = np.stack([_rot(rs) for _ in range(n)])
    t = np.stack([rs.randn(n) * 0.02, rs.randn(n) * 0.02, 0.5 + 0.3 * rs.rand(n)], 1).astype(np.float32)
    K = np.stack([np.array([[110.0 + 10 * rs.rand(), 0, 32 + rs.randn()], [0, 112.0, 31 + rs.randn()], [0, 0, 1]])
                  for _ in range(n)]).astype(np.float32)
    t_true = (t * (1 + rs.uniform(-0.04, 0.04, (n, 1)))).astype(np.float32)
    ids = torch.tensor([models[j].mesh_id for j in mesh_ids], dtype=torch.int32, device=dev)
    sensor = render_meshes(ids, _T(dev, np.concatenate([R, t_true[:, :, None]], 2)), _T(dev, K), 64, 64).cpu().numpy()
    sensor = np.where(rs.rand(n, 64, 64) < 0.9, sensor + 0.002 * rs.randn(n, 64, 64), 0).astype(np.float32)
    xyz = rs.rand(n, 3, 64, 64).astype(np.float32)
    return dict(vf=vf, models=models, mesh_ids=mesh_ids, ids=ids, R=R, t=t, K=K, sensor=sensor, xyz=xyz)


@pytest.mark.gpu
@pytest.mark.parametrize("mask_loss", ["L1", "BCE"])
@pytest.mark.parametrize("coor_z", [False, True])
def test_driver_steps_vs_f64_on_library_renders(dev, coor_z, mask_loss):
    """renderer.depth_refine with iters 1 to 3 over three meshes (mesh_ids): iteration k equals the f64 step fed with
    the library's own render at iteration k-1's translation, which isolates the refine from the rasteriser."""
    from gdrnpp_bop2022_b200.renderer import depth_refine, render_meshes

    d = _driver_case(dev, 11 + 2 * coor_z + (mask_loss == "BCE"))
    n = d["t"].shape[0]
    rs = np.random.RandomState(5)
    mask_mode = 1 if mask_loss == "L1" else 2
    raw = (rs.randn(n, 64, 64) * (2 if mask_mode == 1 else 4)).astype(np.float32)
    args = ([m for m in d["models"]], _T(dev, d["R"]), _T(dev, d["t"]), _T(dev, d["K"]), _T(dev, d["xyz"]),
            _T(dev, raw[:, None]), _T(dev, d["sensor"]))
    t_prev = d["t"]
    skipped = moved = 0
    for k in (1, 2, 3):
        t_k = depth_refine(*args, iters=k, thresh=0.8, mesh_ids=d["mesh_ids"], mask_loss_type=mask_loss,
                           coor_z_refine=coor_z).cpu().numpy()
        ren = render_meshes(d["ids"], _T(dev, np.concatenate([d["R"], t_prev[:, :, None]], 2)), _T(dev, d["K"]), 64, 64)
        ren = ren.cpu().numpy()
        for i in range(n):
            want, st = DO.step(d["xyz"][i], raw[i], ren[i], d["sensor"][i], d["K"][i], t_prev[i], R=d["R"][i],
                               mask_mode=mask_mode, weight_mode=int(coor_z), thresh=0.8, band=DRIVER_BAND)
            ns = st["ns"]
            if ns["sum"] != 0 and (ns["amb"] & (ns["wn"] != 0)).any():
                skipped += 1                          # f32 rounding decides a pixel at the cut: either outcome is right
                continue
            e = np.abs(t_k[i] - want).max() / _ulp32(np.abs(want).max())
            _note("driver_t", e, f"coor_z {coor_z} {mask_loss} iter {k} roi {i}")
            assert e <= BARS["driver_t"][0], (k, i, t_k[i], want, e)
            moved += st["changed"]
        t_prev = t_k
    assert skipped <= 2 and moved >= 2 * n, (skipped, moved)


@pytest.mark.gpu
def test_refine_end_to_end_vs_f64_renders(dev):
    """Two refine iterations over three meshes, each step against the f64 step on f64 renders (raster_oracle) at the
    kernel's translation.  The render's depth error moves only the median: the bar is |ray| * the largest selected
    depth * the render's measured relative depth error on the selected pixels, plus 1 ulp of t.  Pixels the raster
    oracle marks ambiguous take the library's coverage and depth (an f32 rasteriser may decide them either way); those
    ROIs are counted."""
    from gdrnpp_bop2022_b200.renderer import depth_refine, render_meshes
    from oracle import raster_oracle as RO

    d = _driver_case(dev, 21, n=8)
    n = d["t"].shape[0]
    raw = (np.random.RandomState(6).randn(n, 64, 64) * 2).astype(np.float32)
    args = ([m for m in d["models"]], _T(dev, d["R"]), _T(dev, d["t"]), _T(dev, d["K"]), _T(dev, d["xyz"]),
            _T(dev, raw[:, None]), _T(dev, d["sensor"]))
    t_prev, amb_rois = d["t"], 0
    for k in (1, 2):
        t_k = depth_refine(*args, iters=k, thresh=0.8, mesh_ids=d["mesh_ids"]).cpu().numpy()
        ren_lib = render_meshes(d["ids"], _T(dev, np.concatenate([d["R"], t_prev[:, :, None]], 2)), _T(dev, d["K"]), 64, 64)
        ren_lib = ren_lib.cpu().numpy()
        for i in range(n):
            v, f = d["vf"][d["mesh_ids"][i]]
            ro = RO.rasterize(v, f, np.concatenate([d["R"][i], t_prev[i][:, None]], 1), d["K"][i], 64, 64)
            ren64 = ro["depth"].copy()
            amb = ro["ambiguous"]
            if amb.any() and ((ren_lib[i] > 0) | (ren64 > 0))[amb].any():
                amb_rois += 1
                ren64[amb] = ren_lib[i][amb]
            assert np.array_equal(ren64 > 0, ren_lib[i] > 0), (k, i)
            want, st = DO.step(d["xyz"][i], raw[i], ren64.astype(np.float32), d["sensor"][i], d["K"][i], t_prev[i],
                               mask_mode=1, thresh=0.8, band=DRIVER_BAND)
            if st["changed"] and (st["ns"]["amb"] & (st["ns"]["wn"] != 0)).any():
                continue                              # f32 rounding decides a pixel at the cut
            if not st["changed"]:
                assert np.array_equal(t_k[i], t_prev[i]), (k, i)
                continue
            sel = st["ns"]["sel"]
            cov = ren64 > 0
            e_depth = (np.abs(ren_lib[i][cov] - ren64[cov]) / ren64[cov]).max()
            bound = np.abs(st["ray"]) * ren64[sel].max() * (e_depth + 2 * ULP) + _ulp32(want)
            e = (np.abs(t_k[i] - want) / bound).max()
            _note("e2e_t", e, f"iter {k} roi {i}")
            assert e <= BARS["e2e_t"][0], (k, i, t_k[i], want, e)
        t_prev = t_k
    _note("e2e_ambiguous_rois", amb_rois, "")


@pytest.mark.gpu
def test_sensor_crop_kernel_vs_cv2_resize(dev):
    """roi_crop_multi's depth_sensor against cv2.resize(roi_depth, (64, 64)) of the kernel's own 256x256 roi_depth:
    bit-exact with OpenCV's optimised code off, within 2 ulp with it on (the kernel reproduces the unoptimised path)."""
    from test_test_loop import _random_dets, _run_inputs

    rng = np.random.RandomState(4)
    N, H, W = 2, 480, 640
    meta, xywh = _random_dets(rng, N, H, W, 12, 3)
    depth = (rng.randint(300, 3000, (N, H, W)) * (rng.rand(N, H, W) > 0.1)).astype(np.uint16)
    out = _run_inputs(dev, torch.zeros((N, H, W, 3), dtype=torch.uint8, device=dev), meta, xywh,
                      torch.eye(3, device=dev).expand(N, 3, 3).contiguous(), torch.ones((3, 3), device=dev),
                      _T(dev, depth), _T(dev, np.full(N, 1000.0)))
    roi_depth = out["roi_depth"][:, 0].cpu().numpy()
    sensor = out["depth_sensor"].cpu().numpy()
    assert (roi_depth > 0).mean() > 0.1
    assert np.array_equal(sensor.view(np.int32), _cv2_resize(roi_depth, False).view(np.int32))
    fast = _cv2_resize(roi_depth, True)
    assert np.abs(fast.view(np.int32).astype(np.int64) - sensor.view(np.int32).astype(np.int64)).max() <= 2
