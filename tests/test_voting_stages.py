"""The device-side RANSAC voting layer (csrc/ransac_layer.cu: compaction, hypotheses, fused vote + count, winner and
refit) one stage at a time against oracle/voting_oracle.py, a NumPy restatement of the reference driver
(core/csrc/ransac_voting/ransac_voting_gpu.py).

rv_ransac_voting_layer is driven through _lib with a workspace this file allocates, so after a call the compacted
coords / direct and the per-image tn are read out of the workspace at the offsets the C entry carves (base aligned up
to 256 bytes; coords [b,npix,2] f32, direct [b,npix,vn,2] f32, tn [b] i32 padded to 256 bytes, then hypotheses and
counts when the caller passes no buffers of its own).  Every stage is compared with the oracle on the kernel's own
input to that stage:
  * compaction: tn, coords and direct equal the oracle's exactly; a subsampled image keeps a scan-order subsequence of
    its foreground with its own directions, tn within 6 sigma of the binomial mean, the same set for the same seed;
  * hypotheses: bit-exact for caller-supplied pixel pairs (degenerate pairs and zero-norm directions included);
  * counts: equal to the oracle's votes for the layer's own hypotheses (supplied pairs and the device RNG);
  * winner and inlier set: exact (highest count, lowest index on ties, (0, 0) when the best count is 0);
  * refit: within 1 fp32 ulp of the float64 solve on the oracle's inlier set;
  * the batch, the workspace bound, the voting distribution and each entry's mask semantics.

Bars: bit-exact wherever the arithmetic is.  The refit accumulates and solves in float64 and rounds once, so its bar is
1 ulp of the float64 result.  The voting distribution is an fp32 torch computation over hn hypotheses; its bar is
relative to the largest |entry| of each 2x2 covariance and at most 4x the largest error measured.  Measured on an H100
(80GB HBM3, 700 W power limit), with where the largest error occurred, next to each bar below; pytest -s prints them.

Known differences from the reference, pinned here: a subsampled image's kept set depends on its batch index (the
layer's hash draw takes it as input), and so do the device-RNG pixel pairs; an image without foreground enters the
voting distribution with hn = ceil(min_hyp_num / round_hyp_num) * round_hyp_num zero hypotheses, where the reference
emits min_hyp_num of them; a singular refit takes b_inv's identity fallback per keypoint.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import voting_oracle as VO

REFIT_ULP_BAR = 1.0      # 0.4999 ulp  test_counts_exact[33-84-0.999-False], image 0 (the fp32 rounding of the fp64 solve)
DIST_REL_BAR = 2.8e-5    # 7.08e-6     test_voting_distribution_vs_oracle, image 1 (empty: 1024 equal fp32 terms summed)

SENTINEL = 0xA5
GUARD = 512


# ------------------------------------------------------------------------------------------------------------ inputs
def _field(h, w, kps, noise, rs):
    """Unit directions [h,w,vn,2] from every pixel to every keypoint kps [vn,2], with Gaussian noise."""
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    pix = np.stack([xx, yy], -1).astype(np.float64)
    d = np.asarray(kps, np.float64)[None, None] - pix[:, :, None] + rs.randn(h, w, len(kps), 2) * noise
    return (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)


def _disc(h, w, cx, cy, r):
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return ((xx - cx) ** 2 + (yy - cy) ** 2 < r * r).astype(np.float32)


def _pixels(h, w, pts):
    m = np.zeros((h, w), np.float32)
    for x, y in pts:
        m[y, x] = 1
    return m


# ------------------------------------------------------------------------------------------------------ the C entry
class _Run:
    pass


def _run(weights, vertex, hn, thresh=0.999, min_num=5, max_num=30000, seed=1, idxs=None, own_outputs=True, offset=0):
    """One rv_ransac_voting_layer call on a workspace of exactly rv_layer_workspace_bytes(...) bytes, `offset` bytes into a
    256-aligned buffer with SENTINEL guard bytes around it.  own_outputs=False leaves the hypotheses and counts in the
    workspace, where they are read back from."""
    from gdrnpp_bop2022_b200 import _lib

    L = _lib.lib()
    dev = torch.device("cuda:0")
    Wt = torch.from_numpy(np.ascontiguousarray(weights, np.float32)).to(dev)
    Vt = torch.from_numpy(np.ascontiguousarray(vertex, np.float32)).to(dev)
    b, h, w, vn, _ = Vt.shape
    npix = h * w
    nbytes = L.rv_layer_workspace_bytes(b, h, w, vn, hn)
    buf = torch.full((offset + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device=dev)
    assert buf.data_ptr() % 256 == 0
    win = torch.full((b, vn, 2), float("nan"), device=dev)
    hyp = torch.full((b, hn, vn, 2), float("nan"), device=dev) if own_outputs else None
    cnt = torch.full((b, hn, vn), -1, dtype=torch.int32, device=dev) if own_outputs else None
    tn = torch.full((b,), -1, dtype=torch.int32, device=dev)
    inl = torch.zeros((b, vn, npix), dtype=torch.uint8, device=dev)
    ix = None if idxs is None else torch.from_numpy(np.ascontiguousarray(idxs, np.int32)).to(dev)
    _lib.check(L.rv_ransac_voting_layer(_lib.ptr(Wt), _lib.ptr(Vt), b, h, w, vn, hn, float(thresh), int(min_num),
                                        int(max_num), int(seed) & 0xFFFFFFFF, _lib.ptr(ix), _lib.ptr(win), _lib.ptr(hyp),
                                        _lib.ptr(cnt), _lib.ptr(tn), _lib.ptr(inl), ctypes.c_void_p(buf.data_ptr() + offset),
                                        nbytes, _lib.current_stream()), "rv_ransac_voting_layer")
    torch.cuda.synchronize()
    raw = buf.cpu().numpy()
    r = _Run()
    r.guards_intact = bool((raw[:offset] == SENTINEL).all() and (raw[offset + nbytes:] == SENTINEL).all())
    o = (offset + 255) // 256 * 256                          # the carve of rv_ransac_voting_layer

    def take(n, dt, shape, pad=False):
        nonlocal o
        a = raw[o:o + n * 4].copy().view(dt).reshape(shape)
        o += (n * 4 + 255) // 256 * 256 if pad else n * 4
        return a

    r.coords = take(b * npix * 2, np.float32, (b, npix, 2))
    r.direct = take(b * npix * vn * 2, np.float32, (b, npix, vn, 2))
    r.tn_ws = take(b, np.int32, (b,), pad=True)
    hyp_ws = take(b * hn * vn * 2, np.float32, (b, hn, vn, 2))
    cnt_ws = take(b * hn * vn, np.int32, (b, hn, vn))
    assert o <= offset + nbytes
    r.tn = tn.cpu().numpy()
    r.hyp = hyp.cpu().numpy() if own_outputs else hyp_ws
    r.cnt = cnt.cpu().numpy() if own_outputs else cnt_ws
    r.win = win.cpu().numpy()
    r.inl = inl.cpu().numpy()
    return r


_measured = {}


def _note(quantity, err, **case):
    """Keeps the largest error of each quantity and where it occurred."""
    where = os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0].split("::")[-1]
    if err > _measured.get(quantity, (-1.0,))[0]:
        _measured[quantity] = (float(err), where, case)


@pytest.fixture(scope="module", autouse=True)
def _report_measured():
    """Prints the largest refit and distribution errors of the run (pytest -s): the numbers the bars are set from."""
    yield
    for quantity, (err, where, case) in sorted(_measured.items()):
        print("\nvoting stages: largest %s error %.3e at %s %s" % (quantity, err, where, case))


def _ulp_err(got, ref):
    """|got - ref| in fp32 ulps of the float64 result."""
    ref = np.asarray(ref, np.float64)
    return np.abs(np.asarray(got, np.float64) - ref) / np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)


def _check_after_compaction(r, i, coords, direct, thresh, idxs=None):
    """Hypotheses, counts, winner, inlier set and refit of image i, each against the oracle on the kernel's own input
    to that stage.  -> the oracle's stages."""
    tn = coords.shape[0]
    hyp = r.hyp[i]
    if idxs is not None:
        assert np.array_equal(hyp.view(np.uint32), VO.hypotheses(direct, coords, idxs).view(np.uint32))
    cnt = VO.counts(direct, coords, hyp, thresh)
    assert np.array_equal(r.cnt[i], cnt)
    win, idx, best = VO.winner(cnt, hyp)
    inl = VO.inliers(direct, coords, win, thresh)
    assert np.array_equal(r.inl[i, :, :tn], inl)
    assert not r.inl[i, :, tn:].any()
    if tn == 0:
        assert np.array_equal(r.win[i], np.zeros_like(r.win[i]))
        return dict(win=win, idx=idx, best=best, inl=inl, pts=None, singular=None)
    pts, singular = VO.refit(direct, coords, inl)
    err = _ulp_err(r.win[i], pts)
    _note("refit_ulp", err.max(), image=i)
    assert err.max() <= REFIT_ULP_BAR, (i, r.win[i], pts, err)
    return dict(win=win, idx=idx, best=best, inl=inl, pts=pts, singular=singular)


def _check_image(r, i, weights, vertex, thresh, min_num, max_num, idxs=None):
    """Every stage of an image that is not subsampled, from the compaction on."""
    _, coords, direct = VO.compact_image(weights, vertex, min_num, max_num)
    tn = coords.shape[0]
    assert r.tn[i] == tn and r.tn_ws[i] == tn, (i, r.tn[i], r.tn_ws[i], tn)
    assert np.array_equal(r.coords[i, :tn], coords)
    assert np.array_equal(r.direct[i, :tn].view(np.uint32), direct.view(np.uint32))
    return _check_after_compaction(r, i, coords, direct, thresh, idxs)


def _kept(r, i, weights, vertex):
    """The kept set of a subsampled image: a strictly increasing scan-order subsequence of the foreground, each pixel
    with its own directions.  -> (flat pixel indices, coords, direct)."""
    tn = int(r.tn[i])
    assert r.tn_ws[i] == tn
    h, w = weights.shape
    coords, direct = r.coords[i, :tn], r.direct[i, :tn]
    x, y = coords[:, 0].astype(np.int64), coords[:, 1].astype(np.int64)
    assert np.array_equal(coords, np.stack([x, y], 1).astype(np.float32))
    flat = y * w + x
    assert (np.diff(flat) > 0).all() and (flat >= 0).all() and (flat < h * w).all()
    assert (weights.reshape(-1)[flat] != 0).all()
    assert np.array_equal(direct.view(np.uint32), vertex[y, x].view(np.uint32))
    return flat, coords, direct


def _assert_binomial(tn, n_px, fg, max_num):
    sub, p = VO.keep_probability(fg, max_num)
    assert sub
    mean, sd = n_px * p, np.sqrt(n_px * p * (1 - p))
    assert abs(tn - mean) <= 6 * sd, (tn, mean, sd)


def _random_idxs(rs, b, hn, vn):
    return rs.randint(0, 1 << 30, (b, hn, vn, 2)).astype(np.int32)


# ------------------------------------------------------------------------------------------ 1. compaction
@pytest.mark.gpu
def test_compaction_exact_at_the_min_num_edges(dev):
    """Empty, min_num - 1, min_num and ordinary images, and weighted masks (a pixel of weight k counts k times toward
    min_num): tn, coords and direct equal the oracle's; the later stages follow on the same call."""
    rs = np.random.RandomState(0)
    h, w = 37, 53                                              # npix = 1961: not a multiple of 256
    kps = np.array([[20.5, 11.25], [-3.0, 40.0], [70.0, 18.5]])
    corner = [(1, 1), (5, 2), (9, 30), (40, 3), (52, 36)]
    wt = np.stack([np.zeros((h, w), np.float32),
                   _pixels(h, w, corner[:4]),                  # 4 = min_num - 1 pixels: skipped
                   _pixels(h, w, corner),                      # 5 = min_num pixels
                   _disc(h, w, 25, 17, 14),
                   2 * _pixels(h, w, corner[:3]),              # 3 pixels of weight 2: foreground count 6 >= min_num
                   2 * _pixels(h, w, corner[:2]),              # 2 pixels of weight 2: foreground count 4 < min_num
                   _disc(h, w, 20, 20, 9) * (1 + (np.arange(h * w).reshape(h, w) % 3))])   # weights 1..3
    b, hn = wt.shape[0], 64
    vertex = np.stack([_field(h, w, kps, 0.02, rs) for _ in range(b)])
    idxs = _random_idxs(rs, b, hn, len(kps))
    r = _run(wt, vertex, hn, idxs=idxs)
    tns = []
    for i in range(b):
        _check_image(r, i, wt[i], vertex[i], 0.999, 5, 30000, idxs[i])
        tns.append(int(r.tn[i]))
    assert tns[:3] == [0, 0, 5] and tns[4:6] == [3, 0] and tns[3] % 256 != 0


@pytest.mark.gpu
def test_compaction_subsamples_a_vga_image_at_the_default_max_num(dev):
    """A 480 x 640 image with more than 30 000 foreground pixels: the fg > max_num branch keeps a scan-order subsequence,
    about max_num pixels, the same set for the same seed and another for another seed."""
    rs = np.random.RandomState(1)
    h, w = 480, 640
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    mask = (((xx - 320) / 250.0) ** 2 + ((yy - 240) / 200.0) ** 2 < 1).astype(np.float32)
    n_px = int(mask.sum())
    assert n_px > 30000
    v = rs.randn(1, h, w, 2, 2).astype(np.float32)
    a, a2, c = (_run(mask[None], v, 16, seed=s) for s in (7, 7, 8))
    fa, coords, direct = _kept(a, 0, mask, v[0])
    _check_after_compaction(a, 0, coords, direct, 0.999)
    fc, _, _ = _kept(c, 0, mask, v[0])
    _assert_binomial(len(fa), n_px, n_px, 30000)
    _assert_binomial(len(fc), n_px, n_px, 30000)
    assert np.array_equal(a.tn, a2.tn) and np.array_equal(a.coords, a2.coords) and np.array_equal(a.hyp, a2.hyp)
    assert not np.array_equal(fa, fc)


@pytest.mark.gpu
@pytest.mark.parametrize("max_num", [40, 300, 1100])
def test_compaction_subsample_branch_with_small_max_num(dev, max_num):
    """Small max_num values run the subsample branch on a small image, for plain and weighted masks (a weight-2 pixel
    counts twice in the keep probability but is kept or dropped once); every stage after it runs on exactly the kept
    set."""
    rs = np.random.RandomState(max_num)
    h, w = 45, 61
    kps = np.array([[30.2, 22.7], [10.0, 50.5]])
    plain = _disc(h, w, 30, 22, 20)
    weighted = plain * 2
    vertex = np.stack([_field(h, w, kps, 0.05, rs) for _ in range(2)])
    hn = 48
    idxs = _random_idxs(rs, 2, hn, 2)
    wt = np.stack([plain, weighted])
    r = _run(wt, vertex, hn, max_num=max_num, idxs=idxs, seed=max_num)
    n_px = int(plain.sum())
    for i in range(2):
        fg = int(wt[i].sum())
        flat, coords, direct = _kept(r, i, wt[i], vertex[i])
        _assert_binomial(len(flat), n_px, fg, max_num)
        _check_after_compaction(r, i, coords, direct, 0.999, idxs[i])
    r2 = _run(wt, vertex, hn, max_num=max_num, idxs=idxs, seed=max_num)
    r3 = _run(wt, vertex, hn, max_num=max_num, idxs=idxs, seed=max_num + 1)
    assert np.array_equal(r.tn, r2.tn) and np.array_equal(r.coords, r2.coords) and np.array_equal(r.win, r2.win)
    assert not np.array_equal(r.coords[0, :r.tn[0]], r3.coords[0, :r3.tn[0]])


# ------------------------------------------------------------------------------------------ 2. hypotheses
@pytest.mark.gpu
@pytest.mark.parametrize("own_outputs", [True, False])
def test_hypotheses_bit_exact_with_supplied_pairs(dev, own_outputs):
    """Supplied pairs, taken modulo tn, include degenerate pairs (a pixel with itself) and pixels whose direction is
    (0, 0): hypotheses bit-exact against the oracle on the compacted arrays (read from the caller's buffer, or from the
    workspace)."""
    rs = np.random.RandomState(2)
    h, w = 29, 41
    kps = np.array([[14.5, 12.25], [50.0, -5.5], [3.0, 3.0]])
    mask = _disc(h, w, 20, 14, 12)
    vertex = _field(h, w, kps, 0.03, rs)
    zero = rs.rand(h, w) < 0.1
    vertex[zero, 1] = 0.0                                      # zero-norm directions for keypoint 1
    vertex[14, :, 2] = 0.0                                     # and a row of them for keypoint 2
    _, coords, direct = VO.compact_image(mask, vertex, 5, 30000)
    tn, hn, vn = coords.shape[0], 100, 3
    idxs = rs.randint(0, 2 ** 31 - 1, (1, hn, vn, 2)).astype(np.int32)
    idxs[0, :20, :, 1] = idxs[0, :20, :, 0]                    # degenerate pairs
    idxs[0, 20:25, :, 0] = 3
    idxs[0, 20:25, :, 1] = 3 + tn                              # the same pixel after the modulo
    zero_t = np.nonzero((direct[:, 1] == 0).all(-1))[0]
    assert len(zero_t) >= 2
    idxs[0, 30:40, 1, 0] = zero_t[0]
    idxs[0, 30:35, 1, 1] = zero_t[1]                           # both directions zero
    r = _run(mask[None], vertex[None], hn, idxs=idxs, own_outputs=own_outputs)
    _check_image(r, 0, mask, vertex, 0.999, 5, 30000, idxs[0])
    hyp = r.hyp[0]
    assert (hyp[:25] == 0).all() and (hyp[30:40, 1] == 0).all()
    assert (hyp[40:] != 0).any(-1).mean() > 0.7


@pytest.mark.gpu
def test_hypotheses_device_rng_reproducible_per_seed(dev):
    """The device RNG draws the same pixel pairs for the same seed and other pairs for another seed; the counts of its
    hypotheses are the oracle's."""
    rs = np.random.RandomState(3)
    h, w = 33, 47
    kps = np.array([[20.5, 11.25], [40.0, 30.0]])
    mask = _disc(h, w, 23, 16, 13)
    vertex = _field(h, w, kps, 0.03, rs)[None]
    a, a2, c = (_run(mask[None], vertex, 200, seed=s) for s in (11, 11, 12))
    assert np.array_equal(a.hyp.view(np.uint32), a2.hyp.view(np.uint32)) and np.array_equal(a.win, a2.win)
    assert not np.array_equal(a.hyp, c.hyp)
    for r in (a, c):
        _check_image(r, 0, mask, vertex[0], 0.999, 5, 30000)


# ------------------------------------------------------------------------------------------ 3. counts
COUNT_CASES = [  # (hn, vn, thresh, device RNG)
    (1, 9, 0.999, False), (31, 9, 0.99, True), (33, 64, 0.999, False), (33, 1, 0.99, True),
    (257, 9, 0.99, False), (257, 64, 0.999, True), (4096, 1, 0.999, True), (4096, 1, 0.99, False),
    (31, 64, 0.99, False), (33, 84, 0.999, False),     # vn = 84: the largest shared-memory tile
]


@pytest.mark.gpu
def test_count_tile_grows_after_a_smaller_one(dev):
    """The count kernel's shared-memory tile grows with vn (2432 bytes per keypoint).  A call that needs the opt-in
    beyond 48 KB (vn = 21) followed by one at the largest tile (vn = 84) in the same process: the opt-in must cover
    the largest tile, not only the first call's."""
    rs = np.random.RandomState(12)
    h, w = 19, 23
    mask = _disc(h, w, 11, 9, 8)
    for vn in (21, 84, 21):
        kps = np.stack([rs.uniform(0, w, vn), rs.uniform(0, h, vn)], 1)
        vertex = _field(h, w, kps, 0.05, rs)
        r = _run(mask[None], vertex[None], 40, seed=vn)
        _check_image(r, 0, mask, vertex, 0.999, 5, 30000)


@pytest.mark.gpu
@pytest.mark.parametrize("hn,vn,thresh,rng", COUNT_CASES)
def test_counts_exact(dev, hn, vn, thresh, rng):
    """Counts equal the oracle's votes for the layer's own hypotheses, with a tail pixel tile (tn % 256 != 0) and hn
    not a multiple of the 32-hypothesis chunk, for supplied pairs and the device RNG; winner, inliers and refit follow."""
    rs = np.random.RandomState(hn * 100 + vn)
    h, w = 41, 57                                              # npix = 2337
    kps = np.stack([rs.uniform(-10, 67, vn), rs.uniform(-10, 51, vn)], 1)
    wt = np.stack([_disc(h, w, 28, 20, 21), _disc(h, w, 15, 30, 9)])
    vertex = np.stack([_field(h, w, kps, 0.02, rs), _field(h, w, kps, 0.1, rs)])
    idxs = None if rng else _random_idxs(rs, 2, hn, vn)
    r = _run(wt, vertex, hn, thresh=thresh, idxs=idxs, seed=hn + vn)
    for i in range(2):
        assert r.tn[i] % 256 != 0
        _check_image(r, i, wt[i], vertex[i], thresh, 5, 30000, None if rng else idxs[i])


def test_vn_above_the_shared_memory_tile_is_refused_before_any_launch():
    """vn = 85 needs more than the 200 KB shared-memory tile of the count kernel: the entry refuses it before it
    launches anything or touches an output (no GPU needed: nothing runs)."""
    from gdrnpp_bop2022_b200 import _lib

    L = _lib.lib()
    b, h, w, hn = 1, 8, 8, 4
    host = np.zeros(1 << 16, np.float32)
    p = ctypes.c_void_p(host.ctypes.data)
    for vn, refused in ((85, True), (400, True)):
        before = L.gdrn_launch_count()
        nb = L.rv_layer_workspace_bytes(b, h, w, vn, hn)
        rc = L.rv_ransac_voting_layer(p, p, b, h, w, vn, hn, 0.999, 5, 30000, 1, None, p, None, None, None, None, p, nb, None)
        assert (rc != 0) == refused and "shared-memory" in _lib.last_error()
        assert L.gdrn_launch_count() == before and not host.any()


# ------------------------------------------------------------------------------------------ 4. winner and inliers
def _tie_scene():
    """Two 8 x 8 pixel clusters, A pointing at PA and B (A moved 24 pixels right) at PB: a pair inside A gives a
    hypothesis near PA that exactly A's 64 pixels vote for, a pair inside B one near PB with B's 64 votes -- a tie
    between two different points.  Keypoint 3 points every pixel away from PC, so that no hypothesis gets a vote."""
    h, w = 10, 40
    mask = np.zeros((h, w), np.float32)
    mask[:8, :8] = 1
    mask[:8, 24:32] = 1
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    pix = np.stack([xx, yy], -1).astype(np.float64)
    pa, pb, pc = np.array([4.5, 20.25]), np.array([28.5, 20.25]), np.array([20.0, 30.0])
    to = np.where((xx < 16)[:, :, None], pa - pix, pb - pix)
    away = pix - pc
    d = np.stack([to, to, to, away], 2)
    vertex = (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)
    return mask, vertex


def _t(x, y):
    """Compacted index of pixel (x, y) of _tie_scene: 16 foreground pixels per row, A's 8 then B's 8."""
    return y * 16 + (x if x < 8 else 8 + x - 24)


@pytest.mark.gpu
def test_winner_lowest_index_on_ties_across_warps_and_zero_best_count(dev):
    """Ties between different points at hypothesis indices held by different warps of rv_refit_kernel's strided
    arg-max (256 threads; index h is thread h % 256): (5 warp 0, 300 warp 1), (40 warp 1, 261 warp 0: the lower index in
    the higher warp), (5, 261: one thread).  The lowest index must win, which the inlier sets (A's or B's pixels) show.
    Keypoint 3's best count is 0: the winner stays (0, 0), and its inlier set is that of (0, 0)."""
    mask, vertex = _tie_scene()
    hn, vn = 333, 4
    a_pair, b_pair = (_t(0, 0), _t(7, 6)), (_t(24, 0), _t(31, 6))
    idxs = np.zeros((1, hn, vn, 2), np.int32)
    idxs[0, :, :, 1] = idxs[0, :, :, 0] = np.arange(hn)[:, None] % 128   # degenerate pairs: (0, 0), no votes
    for v, (lo, lo_pair, hi, hi_pair) in enumerate([(5, b_pair, 300, a_pair), (40, a_pair, 261, b_pair),
                                                    (5, a_pair, 261, b_pair)]):
        idxs[0, lo, v], idxs[0, hi, v] = lo_pair, hi_pair
    rs = np.random.RandomState(4)
    idxs[0, :, 3, 0] = rs.randint(0, 64, hn) // 8 * 16 + rs.randint(0, 8, hn)          # an A pixel
    idxs[0, :, 3, 1] = rs.randint(0, 64, hn) // 8 * 16 + 8 + rs.randint(0, 8, hn)      # a B pixel
    r = _run(mask[None], vertex[None], hn, idxs=idxs)
    st = _check_image(r, 0, mask, vertex, 0.999, 5, 30000, idxs[0])
    cnt, hyp = r.cnt[0], r.hyp[0]
    for v, (lo, hi) in enumerate([(5, 300), (40, 261), (5, 261)]):
        assert cnt[lo, v] == cnt[hi, v] == cnt[:, v].max() == 64 and (cnt[:, v] == 64).sum() == 2
        assert not np.array_equal(hyp[lo, v], hyp[hi, v])
        assert st["idx"][v] == lo
    in_a = (r.coords[0, :r.tn[0], 0] < 16)
    assert np.array_equal(r.inl[0, 0, :128].astype(bool), ~in_a)                      # B won at index 5
    assert np.array_equal(r.inl[0, 1, :128].astype(bool), in_a)                       # A won at index 40
    assert np.array_equal(r.inl[0, 2, :128].astype(bool), in_a)                       # A won at index 5
    assert cnt[:, 3].max() == 0 and (hyp[:, 3] != 0).all()
    assert np.array_equal(st["win"][3], [0, 0]) and r.inl[0, 3].sum() >= 2            # inliers of (0, 0) ...
    assert np.abs(r.win[0, 3] - [20.0, 30.0]).max() < 1e-3                            # ... whose lines meet at PC


# ------------------------------------------------------------------------------------------ 5. refit
@pytest.mark.gpu
def test_refit_singular_systems_take_the_identity_fallback(dev):
    """Every inlier line of the winner parallel (collinear pixels sharing one direction, their hypothesis made by two
    pixels that point away from it and so do not vote): ATA is singular and the refit returns ATb, b_inv's identity
    fallback -- once with axis-aligned lines (ATA exactly singular), once along (0.6, 0.8)."""
    h, w = 40, 50
    mask = np.zeros((h, w), np.float32)
    vertex = np.zeros((h, w, 2, 2), np.float32)
    p0, p1 = np.array([30.0, 5.0]), np.array([36.0, 48.0])
    row = [(x, 5) for x in range(20)]                           # on y = 5, pointing at p0 along +x
    diag = [(3 * k, 4 * k) for k in range(1, 9)]                # on y = 4/3 x, pointing at p1 along (0.6, 0.8)
    q = [(35, 0), (35, 9), (40, 30), (30, 39)]
    for x, y in row + diag + q:
        mask[y, x] = 1
    for x, y in row:
        vertex[y, x, 0] = (1.0, 0.0)
    for x, y in diag:
        vertex[y, x, 1] = (0.6, 0.8)
    for x, y in q:                                              # lines through p0 / p1, pointing away from them
        for v, p in enumerate((p0, p1)):
            d = np.array([x, y], np.float64) - p
            vertex[y, x, v] = d / np.linalg.norm(d)
    _, coords, direct = VO.compact_image(mask, vertex, 5, 30000)
    t = {(int(cx), int(cy)): k for k, (cx, cy) in enumerate(coords)}
    hn = 8
    idxs = np.zeros((1, hn, 2, 2), np.int32)
    idxs[0, :, 0] = (t[q[0]], t[q[1]])
    idxs[0, :, 1] = (t[q[2]], t[q[3]])
    r = _run(mask[None], vertex[None], hn, idxs=idxs)
    st = _check_image(r, 0, mask, vertex, 0.999, 5, 30000, idxs[0])
    assert st["singular"].all()
    assert st["inl"][0].sum() == len(row) and st["inl"][1].sum() == len(diag)
    assert np.array_equal(r.win[0, 0], [0.0, 100.0])            # ATb: normals (0, -1), b = -5, twenty of them
    _, atb = VO.normal_equations(direct, coords, st["inl"])
    assert (_ulp_err(r.win[0], atb) <= REFIT_ULP_BAR).all()


# ------------------------------------------------------------------------------------------ 6. batch
@pytest.mark.gpu
def test_batch_of_every_kind_of_image(dev):
    """One call over an empty image, one below min_num, one at min_num, an ordinary one and a subsampled one.  Every image
    that is not subsampled is bit-identical alone and inside the batch.  A subsampled image's kept set is drawn by a
    hash of (seed, batch index, pixel): alone (index 0) and at index 4 it is a different draw, each a valid one."""
    rs = np.random.RandomState(6)
    h, w = 48, 56
    kps = np.array([[24.5, 20.0], [60.0, 5.5], [10.0, 40.0]])
    corner = [(0, 0), (10, 3), (55, 47), (30, 30), (2, 40)]
    wt = np.stack([np.zeros((h, w), np.float32), _pixels(h, w, corner[:4]), _pixels(h, w, corner),
                   _disc(h, w, 25, 22, 15), _disc(h, w, 28, 24, 24)])
    max_num = 1000
    assert wt[3].sum() < max_num < wt[4].sum()
    b, hn, vn = 5, 96, 3
    vertex = np.stack([_field(h, w, kps, 0.03, rs) for _ in range(b)])
    idxs = _random_idxs(rs, b, hn, vn)
    r = _run(wt, vertex, hn, max_num=max_num, idxs=idxs, seed=21)
    for i in range(4):
        _check_image(r, i, wt[i], vertex[i], 0.999, 5, max_num, idxs[i])
        alone = _run(wt[i:i + 1], vertex[i:i + 1], hn, max_num=max_num, idxs=idxs[i:i + 1], seed=21)
        tn = int(r.tn[i])
        assert alone.tn[0] == tn
        for name in ("coords", "direct"):
            assert np.array_equal(getattr(alone, name)[0, :tn].view(np.uint8), getattr(r, name)[i, :tn].view(np.uint8))
        for name in ("hyp", "cnt", "win", "inl"):
            assert np.array_equal(getattr(alone, name)[0].view(np.uint8), getattr(r, name)[i].view(np.uint8)), name
    flat_b, coords, direct = _kept(r, 4, wt[4], vertex[4])
    _check_after_compaction(r, 4, coords, direct, 0.999, idxs[4])
    alone = _run(wt[4:], vertex[4:], hn, max_num=max_num, idxs=idxs[4:], seed=21)
    flat_a, coords, direct = _kept(alone, 0, wt[4], vertex[4])
    _check_after_compaction(alone, 0, coords, direct, 0.999, idxs[4])
    n_px = int(wt[4].sum())
    _assert_binomial(len(flat_a), n_px, n_px, max_num)
    _assert_binomial(len(flat_b), n_px, n_px, max_num)
    assert not np.array_equal(flat_a, flat_b)                   # the batch index is an input of the draw


# ------------------------------------------------------------------------------------------ 7. workspace
@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 3, 64, 65])
def test_workspace_of_exactly_the_reported_size(dev, b):
    """A workspace of exactly rv_layer_workspace_bytes(...) bytes at base offsets 0, 4 and 252 of a 256-aligned buffer
    (the carve aligns the base up to 256 bytes and pads the tn block to 256: b = 64 fills it, 65 spills into a second
    block), with the hypotheses and counts in the caller's buffers or in the workspace: nothing is written outside it,
    and every output is bit-identical to the first call's."""
    rs = np.random.RandomState(b)
    h, w, vn, hn = 13, 21, 3, 37
    kps = np.array([[10.5, 6.25], [-4.0, 20.0], [30.0, 0.5]])
    wt = np.stack([_disc(h, w, 10, 6, 3 + (i % 5)) for i in range(b)])
    vertex = np.stack([_field(h, w, kps, 0.05, rs) for _ in range(b)])
    idxs = _random_idxs(rs, b, hn, vn)
    base = None
    for own in (True, False):
        for offset in (0, 4, 252):
            r = _run(wt, vertex, hn, idxs=idxs, own_outputs=own, offset=offset)
            assert r.guards_intact, (own, offset)
            if base is None:
                base = r
                for i in range(min(b, 4)):
                    _check_image(r, i, wt[i], vertex[i], 0.999, 5, 30000, idxs[i])
                continue
            for name in ("tn", "tn_ws", "hyp", "cnt", "win", "inl"):
                got, ref = getattr(r, name), getattr(base, name)
                assert np.array_equal(got.view(np.uint8), ref.view(np.uint8)), (own, offset, name)
            for i in range(b):
                tn = int(base.tn[i])
                assert np.array_equal(r.coords[i, :tn], base.coords[i, :tn])
                assert np.array_equal(r.direct[i, :tn].view(np.uint32), base.direct[i, :tn].view(np.uint32))


# ------------------------------------------------------------------------------------------ 8. voting distribution
@pytest.mark.gpu
def test_voting_distribution_vs_oracle(dev):
    """estimate_voting_distribution_with_mean against the float64 oracle on the layer's own hypotheses, counts and tn
    (the same seed through _ransac_layer_call).  The mask holds 0, 1, 2 and 0.5, so only `mask == 1` is foreground;
    min_hyp_num = 1000 with rounds of 256 gives hn = 1024.  Image 1 is empty: it takes the ratio-of-1 rule with hn zero
    hypotheses (the reference emits min_hyp_num = 1000 of them; the covariances differ by a factor
    1000 * 1024.001 / (1024 * 1000.001), 1 - 2e-8)."""
    from gdrnpp_bop2022_b200.native_ops import _ransac_layer_call, estimate_voting_distribution_with_mean

    rs = np.random.RandomState(8)
    h, w = 50, 66
    kps = np.array([[30.5, 20.25], [70.0, 40.0], [5.0, -8.0]])
    fg = _disc(h, w, 33, 25, 20)
    mask = np.stack([fg + (rs.rand(h, w) < 0.3) * fg, np.zeros((h, w), np.float32),
                     fg * np.where(rs.rand(h, w) < 0.5, 1.0, 0.5), fg])
    b, vn = mask.shape[0], len(kps)
    vertex = np.stack([_field(h, w, kps, n, rs) for n in (0.02, 0.02, 0.05, 0.3)])
    M, V = torch.from_numpy(mask.astype(np.float32)).to(dev), torch.from_numpy(vertex).to(dev)
    mean = torch.from_numpy(np.tile(kps, (b, 1, 1)).astype(np.float32) + rs.randn(b, vn, 2).astype(np.float32)).to(dev)
    m2, cov = estimate_voting_distribution_with_mean(M, V, mean, round_hyp_num=256, min_hyp_num=1000, inlier_thresh=0.99,
                                                     seed=31)
    _, hyp, cnt, tn, _ = _ransac_layer_call(M == 1, V, 1024, 0.99, 5, 30000, None, 31, want_hyp=True)
    torch.cuda.synchronize()
    hyp, cnt, tn = hyp.cpu().numpy(), cnt.cpu().numpy(), tn.cpu().numpy()
    assert torch.equal(m2, mean) and hyp.shape[1] == 1024
    assert list(tn) == [int((mask[i] == 1).sum()) for i in range(b)] and tn[0] < int((mask[0] != 0).sum())
    assert not hyp[1].any() and not cnt[1].any()
    ref = VO.voting_distribution(hyp, cnt, tn, mean.cpu().numpy())
    got = cov.cpu().numpy().astype(np.float64)
    rel = np.abs(got - ref).max((2, 3)) / np.abs(ref).max((2, 3))
    _note("dist_rel", rel.max(), at=np.unravel_index(rel.argmax(), rel.shape))
    assert rel.max() <= DIST_REL_BAR, rel


@pytest.mark.gpu
def test_voting_distribution_drop_boundary_and_normaliser(dev):
    """The covariance step on constructed hypotheses and counts: a ratio exactly at max - 0.1 (9 / 10 = 0.9f = 1.0f -
    0.1f) is kept and one below it dropped; a keypoint whose only non-zero ratio is 0.1 makes the + 1e-3 normaliser a
    1 % term; an image with tn = 0 weighs its zero hypotheses by 1."""
    from gdrnpp_bop2022_b200.native_ops import _voting_distribution

    hn, vn = 40, 3
    rs = np.random.RandomState(9)
    hyp = rs.uniform(-50, 50, (2, hn, vn, 2)).astype(np.float32)
    cnt = np.zeros((2, hn, vn), np.int32)
    tn = np.array([10, 0], np.int32)
    cnt[0, :, 0] = rs.choice([10, 9, 8, 3], hn)                 # ratios 1, 0.9 (kept: the boundary), 0.8, 0.3 (dropped)
    cnt[0, :4, 0] = (10, 9, 8, 9)
    cnt[0, :, 1] = 0
    cnt[0, 7, 1] = 1                                            # tn = 10 -> ratio 0.1, alone: normaliser 0.1 + 1e-3
    cnt[0, :, 2] = rs.randint(0, 11, hn)
    hyp[1] = 0.0
    mean = rs.uniform(-5, 5, (2, vn, 2)).astype(np.float32)
    T = lambda a: torch.from_numpy(a).to(dev)
    got = _voting_distribution(T(hyp), T(cnt), T(tn), T(mean)).cpu().numpy().astype(np.float64)
    ref = VO.voting_distribution(hyp, cnt, tn, mean)
    rel = np.abs(got - ref).max((2, 3)) / np.abs(ref).max((2, 3))
    _note("dist_rel", rel.max(), at=np.unravel_index(rel.argmax(), rel.shape))
    assert rel.max() <= DIST_REL_BAR, rel
    # the boundary decides: dropping the ratio-0.9 hypotheses, or keeping the 0.8 ones, moves the covariance far
    for alt in (np.where(cnt[0, :, 0] == 9, 0, cnt[0, :, 0]), np.where(cnt[0, :, 0] == 8, 9, cnt[0, :, 0])):
        c2 = cnt.copy()
        c2[0, :, 0] = alt
        moved = VO.voting_distribution(hyp, c2, tn, mean)[0, 0]
        assert np.abs(moved - ref[0, 0]).max() > 100 * DIST_REL_BAR * np.abs(ref[0, 0]).max()
    # tn = 0: hn hypotheses at zero, each weighed 1
    m = mean[1].astype(np.float64)
    assert np.allclose(ref[1], hn / (hn + 1e-3) * m[:, :, None] * m[:, None, :], rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------ 9. mask semantics
@pytest.mark.gpu
def test_mask_semantics_of_each_entry(dev):
    """ransac_voting_layer reads a byte mask as its reference does (`.byte()`): a value in (0, 1) is background, a pixel
    of value k counts k times toward min_num, max_num and the keep probability.  ransac_voting_layer_v3 reads a bool
    mask (`.to(torch.bool)`): every non-zero value is one pixel.  Image 0: values 0.5, 1 and 1.7; image 1: three pixels
    of value 2 (6 >= min_num under v1, 3 < min_num under v3); image 2: 600 pixels of value 2 at max_num = 1000
    (subsampled under v1, not under v3)."""
    from gdrnpp_bop2022_b200.native_ops import ransac_voting_layer, ransac_voting_layer_v3

    rs = np.random.RandomState(10)
    h, w = 40, 50
    kps = np.array([[25.5, 18.25], [60.0, 10.0]])
    img0 = _disc(h, w, 25, 20, 16) * rs.choice([0.5, 1.0, 1.7], (h, w))
    img1 = 2 * _pixels(h, w, [(3, 3), (20, 30), (45, 5)])
    img2 = np.zeros((h, w), np.float32)
    img2[5:35, 10:30] = 2.0
    mask = np.stack([img0, img1, img2]).astype(np.float32)
    vertex = np.stack([_field(h, w, kps, 0.03, rs) for _ in range(3)])
    hn, max_num = 80, 1000
    idxs = _random_idxs(rs, 3, hn, 2)
    M, V, I = (torch.from_numpy(a).to(dev) for a in (mask, vertex, idxs))
    for fn, sem in ((ransac_voting_layer, "byte"), (ransac_voting_layer_v3, "bool")):
        win, inl, tn = (t.cpu().numpy() for t in fn(M, V, hn, max_num=max_num, idxs=I, return_inliers=True, seed=5))
        wts = VO.foreground_weights(mask, sem)
        for i in range(3):
            n_px, fgw = int((wts[i] != 0).sum()), int(wts[i].sum())
            if VO.keep_probability(fgw, max_num)[0]:
                assert sem == "byte" and i == 2
                _assert_binomial(int(tn[i]), n_px, fgw, max_num)
                continue
            ref = VO.voting_layer(wts[i], vertex[i], idxs[i], 0.999, 5, max_num)
            assert tn[i] == ref["tn"], (sem, i)
            assert np.array_equal(inl[i, :, :ref["tn"]], ref["inliers"])
            if ref["tn"]:
                assert (_ulp_err(win[i], ref["pts"]) <= REFIT_ULP_BAR).all()
            else:
                assert not win[i].any()
        expect = {"byte": [int((np.trunc(img0) != 0).sum()), 3], "bool": [int((img0 != 0).sum()), 0]}[sem]
        assert list(tn[:2]) == expect and (sem == "byte") == (tn[2] < 600)


# ------------------------------------------------------------------------------------------ the oracle itself (CPU)
def test_oracle_refit_hand_worked():
    """Lines y = 0 (pixel (0, 0), direction (1, 0)) and x = 3 (pixel (3, 4), direction (0, 1)) meet at (3, 0); the
    three-line system with (6, 2) pointing along (-1, -1) / sqrt 2 at (4, 0) is the least-squares point of its normals."""
    coords = np.array([[0, 0], [3, 4]], np.float32)
    direct = np.array([[[1, 0]], [[0, 1]]], np.float32)
    pts, singular = VO.refit(direct, coords, np.ones((1, 2), np.uint8))
    assert not singular[0] and np.allclose(pts[0], [3, 0], atol=1e-15)
    s = np.float32(1 / np.sqrt(2))
    coords = np.array([[0, 0], [3, 4], [6, 2]], np.float32)
    direct = np.array([[[1, 0]], [[0, 1]], [[-s, -s]]], np.float32)
    pts, _ = VO.refit(direct, coords, np.ones((1, 3), np.uint8))
    n = np.array([[0, -1], [1, 0], [-s, s]], np.float64)
    b = (n * coords).sum(1)
    assert np.allclose(pts[0], np.linalg.lstsq(n, b, rcond=None)[0], rtol=0, atol=1e-12)
    inl = np.array([[1, 1, 0]], np.uint8)                      # the inlier mask selects the lines
    assert np.allclose(VO.refit(direct, coords, inl)[0][0], [3, 0], atol=1e-15)


def test_oracle_refit_singular_takes_the_identity_fallback():
    """Parallel lines y = 1 and y = 2 (directions (1, 0)): ATA = diag(0, 2) is singular and the result is ATb =
    (0, 1 + 2); with no inliers at all it is (0, 0)."""
    coords = np.array([[0, 1], [5, 2]], np.float32)
    direct = np.array([[[1, 0]], [[-1, 0]]], np.float32)
    pts, singular = VO.refit(direct, coords, np.ones((1, 2), np.uint8))
    assert singular[0] and np.array_equal(pts[0], [0.0, 1.0 + 2.0])
    pts, singular = VO.refit(direct, coords, np.zeros((1, 2), np.uint8))
    assert singular[0] and np.array_equal(pts[0], [0.0, 0.0])


def test_oracle_winner_rule():
    """Highest count, lowest index on ties, (0, 0) when the best count is 0."""
    cnt = np.array([[3, 0], [7, 0], [7, 0], [1, 0]])
    hyp = np.arange(16, dtype=np.float32).reshape(4, 2, 2) + 1
    win, idx, best = VO.winner(cnt, hyp)
    assert list(idx) == [1, 0] and list(best) == [7, 0]
    assert np.array_equal(win, [hyp[1, 0], [0, 0]])


def test_oracle_voting_distribution_hand_worked():
    """tn = 10, counts 10, 9, 8 at (1, 0), (0, 2), (3, 3) around (0, 0): ratios 1, 0.9 (= 1.0f - 0.1f, kept) and 0.8
    (dropped) -> [[1, 0], [0, 0.9 * 4]] / (1.9 + 1e-3); an empty image weighs its zero hypotheses by 1."""
    hyp = np.array([[[[1, 0]], [[0, 2]], [[3, 3]]]], np.float32)
    cnt = np.array([[[10], [9], [8]]])
    cov = VO.voting_distribution(hyp, cnt, np.array([10]), np.zeros((1, 1, 2)))
    r9 = np.float64(np.float32(0.9))
    assert np.allclose(cov[0, 0], np.array([[1, 0], [0, 4 * r9]]) / (1 + r9 + 1e-3), rtol=1e-15, atol=0)
    m = np.array([[[2.0, -1.0]]])
    cov = VO.voting_distribution(np.zeros((1, 3, 1, 2), np.float32), np.zeros((1, 3, 1)), np.array([0]), m)
    assert np.allclose(cov[0, 0], 3 / (3 + 1e-3) * np.outer(m[0, 0], m[0, 0]), rtol=1e-15, atol=0)


def test_oracle_mask_semantics_and_compaction_order():
    """Byte, bool and == 1 readings of one mask; compaction in row-major order with (x, y) coordinates."""
    mask = np.array([[0, 0.5, 1], [1.7, 2, 3.9]], np.float32)
    assert VO.foreground_weights(mask, "byte").tolist() == [[0, 0, 1], [1, 2, 3]]
    assert VO.foreground_weights(mask, "bool").tolist() == [[0, 1, 1], [1, 1, 1]]
    assert VO.foreground_weights(mask, "eq1").tolist() == [[0, 0, 1], [0, 0, 0]]
    vertex = np.arange(12, dtype=np.float32).reshape(2, 3, 1, 2)
    fg, coords, direct = VO.compact_image(VO.foreground_weights(mask, "byte"), vertex, 5, 30000)
    assert fg == 7 and coords.tolist() == [[2, 0], [0, 1], [1, 1], [2, 1]]
    assert np.array_equal(direct, vertex.reshape(6, 1, 2)[[2, 3, 4, 5]])
    assert VO.compact_image(VO.foreground_weights(mask, "bool"), vertex, 5, 30000)[0] == 5
    assert VO.compact_image(VO.foreground_weights(mask, "eq1"), vertex, 5, 30000)[1].shape == (0, 2)
    assert VO.keep_probability(1200, 1000) == (True, float(np.float32(1000) / np.float32(1200)))
    assert VO.keep_probability(1000, 1000) == (False, 1.0)
