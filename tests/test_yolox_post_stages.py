"""YOLOX post-process one stage at a time against the NumPy oracle (oracle/yolox_post_oracle.py) and torchvision.

csrc/yolox_post.cu leaves every stage's result in its workspace (yolox_postprocess_layout gives the offsets): the
compacted decoded rows, the scores, the rank order, the candidate count, the largest coordinate and the NMS bit masks.
Each stage is checked on the kernel's own input to it, so an error upstream can neither hide nor leak into a later
check: decode and the filter bit-exact against the fp32 replica (w, h within expf's 2 ulp of fp64), the rank order
exactly, every mask word exactly, and the greedy reduce against a pass over the kernel's own masks.  The NMS is then
compared end to end with torchvision's batched_nms / nms on CUDA, including both sides of its 25 000-candidate switch,
and the keep-single-instance path (csrc/yolox_net.cu) with torchvision's CPU nms, which is what the reference runs.

Every GPU case runs its call twice and requires bit-identical results.  The oracle-pinning tests at the top need no
GPU.
"""
import numpy as np
import pytest
import torch

from oracle import yolox_post_oracle as P

F32 = np.float32
NC = 21
HW_SHIPPED, STRIDES = [(80, 80), (40, 40), (20, 20)], [8, 16, 32]
TTA_SCALES = (1, 0.75, 0.83, 1.12, 1.25)


def tta_levels():
    """The levels of the shipped test-time augmentation at 640 x 640: 43 428 anchors."""
    hw, st = [], []
    for s in TTA_SCALES:
        side = -(-int(640 * s) // 32) * 32 if s != 1 else 640
        hw += [(side // k, side // k) for k in STRIDES]
        st += STRIDES
    return hw, st


# ---------------------------------------------------------------------------------------------------------------------
# oracle pinning (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def midpoint_fma_cases():
    """(x, y, z) whose fp64 sum x * y + z lands on an fp32 midpoint while the exact one does not: x * y = 2^-24 (1 + d)
    with 0 < |d| < 2^-29 and z = 1 (sum on 1 + 2^-24) or z = +-(1 + 2^-23) (sums on 1 + 3 2^-24 and
    -(1 + 2^-24)), where ties-to-even of the fp64 sum goes the wrong way."""
    out = []
    for m in range(1, 1 << 16):
        x = F32(1 + m * 2.0 ** -23)
        y = F32(F32(1.0) / x)
        for yy in (y, np.nextafter(y, F32(2)), np.nextafter(y, F32(0))):
            d = float(x) * float(yy) - 1.0
            if 0 < abs(d) < 2.0 ** -29:
                out += [(x, F32(yy * F32(2.0 ** -24)), z) for z in (F32(1), F32(1 + 2.0 ** -23), F32(-1 - 2.0 ** -23))]
        if len(out) >= 48:
            break
    return out


def test_fma_emulation_matches_exact_rationals():
    rng = np.random.default_rng(0)
    x = rng.uniform(0.5, 300, 3000).astype(F32)
    y = rng.uniform(0.5, 300, 3000).astype(F32)
    z = (rng.uniform(-1, 1, 3000) * 9e4).astype(F32)
    got = P.fma_f32(x, y, z)
    assert all(got[i] == P.fma_f32_fraction(x[i], y[i], z[i]) for i in range(len(x)))
    cases = midpoint_fma_cases()
    assert len(cases) >= 8
    naive_wrong = 0
    for x, y, z in cases:
        exact = P.fma_f32_fraction(x, y, z)
        s64 = float(x) * float(y) + float(z)
        r = F32(s64)
        other = np.nextafter(r, F32(np.inf) if s64 > float(r) else F32(-np.inf))
        assert s64 != float(r) and abs(s64 - float(r)) == abs(float(other) - s64)   # on an fp32 midpoint
        assert P.fma_f32(x, y, z) == exact, (x, y, z)
        naive_wrong += F32(s64) != exact
    assert naive_wrong > 0   # some of them are the ones plain double rounding gets wrong


def test_oracle_nms_matches_torchvision_cpu():
    """torchvision's CPU nms and both batched paths, called directly, against the oracle's CPU arithmetic on clustered
    boxes with planted near-threshold pairs (distinct scores: the vanilla path's final sort is not stable)."""
    tv = pytest.importorskip("torchvision")
    from torchvision.ops import boxes as TB

    rng = np.random.default_rng(1)
    for thr in (0.65, 0.3, 0.45):
        pa, pb = P.near_threshold_pairs(rng, 60, thr, span=6)
        sel = rng.choice(len(pa), 80, replace=False)
        boxes = np.concatenate([P.xyxy(*pa[sel].T), P.xyxy(*pb[sel].T), cluster_boxes(rng, 150)]).astype(F32)
        n = len(boxes)
        scores = rng.permutation(n).astype(F32) / F32(n) + F32(0.01)
        cls = rng.integers(0, 4, n)
        bt, st, ct = torch.from_numpy(boxes), torch.from_numpy(scores), torch.from_numpy(cls)
        assert np.array_equal(tv.ops.nms(bt, st, thr).numpy(), P.nms(boxes, scores, thr, "cpu"))
        assert np.array_equal(TB._batched_nms_coordinate_trick(bt, st, ct, thr).numpy(),
                              P.batched_nms_trick(boxes, scores, cls, thr, "cpu"))
        assert np.array_equal(TB._batched_nms_vanilla(bt, st, ct, thr).numpy(),
                              P.batched_nms_vanilla(boxes, scores, cls, thr, "cpu"))
        # tied scores: nms sorts stably, lower index first
        tied = (np.round(scores * 4) / 4).astype(F32)
        assert np.array_equal(tv.ops.nms(bt, torch.from_numpy(tied), thr).numpy(), P.nms(boxes, tied, thr, "cpu"))


def test_oracle_hand_worked_cases():
    tv = pytest.importorskip("torchvision")
    from torchvision.ops import boxes as TB

    def both(boxes, thr, form, cls=None):
        b = np.asarray(boxes, F32)
        s = np.array([0.9, 0.8], F32)
        if cls is None:
            return P.nms(b, s, thr, form)
        return P.batched_nms_trick(b, s, np.asarray(cls), thr, form)

    # IoU exactly 0.5 at thr 0.5 is kept (IoU > thr suppresses), in every form
    half = [[0, 0, 4, 1], [0, 0, 2, 1]]
    assert P.iou64(*np.array(half, F32)) == 0.5
    for form in ("cuda", "cpu"):
        assert both(half, 0.5, form).tolist() == [0, 1]
    assert tv.ops.nms(torch.tensor(half, dtype=torch.float32), torch.tensor([0.9, 0.8]), 0.5).tolist() == [0, 1]
    # fp32 IoU == float32(0.3): the CPU compares with the double 0.3 (suppresses), CUDA with float32(0.3) (keeps)
    b3 = [[0, 0, 10, 10], [0, 0, 3, 10]]
    assert P.iou_cpu_f32(*np.array(b3, F32)) == F32(0.3) and P.iou64(*np.array(b3, F32)) == 0.3
    assert both(b3, 0.3, "cpu").tolist() == [0] and both(b3, float(F32(0.3)), "cpu").tolist() == [0, 1]
    assert both(b3, 0.3, "cuda").tolist() == [0, 1]
    assert tv.ops.nms(torch.tensor(b3, dtype=torch.float32), torch.tensor([0.9, 0.8]), 0.3).tolist() == [0]
    # two zero-area boxes: 0 / 0 is nan and suppresses nothing
    z = [[5, 5, 5, 5], [5, 5, 5, 5]]
    assert np.isnan(P.iou_cuda_f32(*np.array(z, F32))) and np.isnan(P.iou_cpu_f32(*np.array(z, F32)))
    for form in ("cuda", "cpu"):
        assert both(z, 0.1, form).tolist() == [0, 1]
    assert tv.ops.nms(torch.tensor(z, dtype=torch.float32), torch.tensor([0.9, 0.8]), 0.1).tolist() == [0, 1]
    # negative coordinates: the coordinate trick lets class 1 suppress class 0 (max -10 -> class 1 shifted by -9)
    neg, ncls = [[-95, -95, -10, -10], [-100, -100, -10, -10]], [1, 0]
    assert P.trick_offsets(np.array(neg, F32), ncls)[0].tolist() == [-9.0, 0.0]
    assert both(neg, 0.5, "cuda", ncls).tolist() == [0] and both(neg, 0.5, "cpu", ncls).tolist() == [0]
    got = TB._batched_nms_coordinate_trick(torch.tensor(neg, dtype=torch.float32), torch.tensor([0.9, 0.8]), torch.tensor(ncls), 0.5)
    assert got.tolist() == [0]
    assert TB._batched_nms_vanilla(torch.tensor(neg, dtype=torch.float32), torch.tensor([0.9, 0.8]), torch.tensor(ncls), 0.5).tolist() == [0, 1]


def test_oracle_keep_single_instance_matches_host_restatement():
    """The fp32 keep-single-instance oracle against the fp64 host restatement (oracle/yolox_oracle.py) away from the
    thresholds: same classes, same rows to fp32 rounding."""
    from oracle import yolox_oracle as O

    rng = np.random.default_rng(2)
    for nc in (1, 3, 8):
        for _ in range(20):
            d = random_dec(rng, 60, nc)
            ious = []
            ref = O.keep_single_instance(d, nc, 0.3, 0.45, ious=ious)
            if any(abs(i - 0.45) < 1e-4 for i in ious):
                continue
            _, rows = P.keep_single_instance(d, nc, 0.3, 0.45)
            if ref is None:
                assert len(rows) == 0
                continue
            assert rows.shape == ref.shape
            assert np.abs(rows.astype(np.float64) - ref).max() < 1e-3


def test_oracle_stage_helpers():
    # class max: the first maximum
    cc, cp = P.class_max(np.array([[0.2, 0.7, 0.7], [0.5, 0.5, 0.1], [0, 0, 0]], F32))
    assert cp.tolist() == [1, 0, 0] and torch.max(torch.tensor([[0.2, 0.7, 0.7], [0.5, 0.5, 0.1]]), 1)[1].tolist() == [1, 0]
    # filter: score = obj * cls in fp32 against float32(conf); the band is where rounding decides
    conf = 0.3
    s32, k32, k64 = P.score_filter(np.ones(3, F32), np.array([np.nextafter(F32(conf), F32(0)), F32(conf),
                                                              np.nextafter(F32(conf), F32(1))]), conf)
    assert k32.tolist() == [False, True, True] and k64.tolist() == [False, True, True]
    s32, k32, k64 = P.score_filter(np.ones(1, F32), np.array([F32(0.65)]), 0.65)   # 0.65 rounds down in fp32
    assert k32.tolist() == [True] and k64.tolist() == [False]
    # rank: stable
    assert P.rank(np.array([0.5, 0.7, 0.5, 0.7], F32)).tolist() == [1, 3, 0, 2]
    # mask words round trip through the greedy pass
    rng = np.random.default_rng(3)
    sup = np.triu(rng.random((150, 150)) < 0.05, 1)
    assert np.array_equal(P.greedy_words(P.mask_words(sup), 150), P.greedy(sup))
    # planted pairs straddle the threshold
    pa, pb = P.near_threshold_pairs(rng, 50, 0.65)
    i64 = P.iou64(P.xyxy(*pa.T), P.xyxy(*pb.T))
    assert (i64 > 0.65).any() and (i64 < 0.65).any() and np.abs(i64 - 0.65).max() < 1e-3


# ---------------------------------------------------------------------------------------------------------------------
# shared builders
# ---------------------------------------------------------------------------------------------------------------------
def cluster_boxes(rng, n, centre_lo=60.0, centre_hi=560.0, k=6):
    """xyxy fp32 boxes jittered around k cluster centres (many overlapping pairs)."""
    c = rng.uniform(centre_lo, centre_hi, (k, 2))
    pick = rng.integers(0, k, n)
    cxy = c[pick] + rng.normal(0, 8, (n, 2))
    wh = rng.uniform(30, 90, (n, 2))
    return P.xyxy(cxy[:, 0], cxy[:, 1], wh[:, 0], wh[:, 1])


def to_cxcywh(b):
    """xyxy -> cxcywh fp32 (only used for boxes whose corners then decode exactly: integer-ish sizes)."""
    b = np.asarray(b, np.float64)
    return np.stack([(b[:, 0] + b[:, 2]) / 2, (b[:, 1] + b[:, 3]) / 2, b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]], 1).astype(F32)


def random_dec(rng, A, nc):
    d = np.zeros((A, 5 + nc), F32)
    d[:, 0:2] = rng.uniform(40, 600, (A, 2))
    d[:, 2:4] = rng.uniform(10, 120, (A, 2))
    d[:, 4] = rng.random(A)
    d[:, 5:] = rng.random((A, nc)) ** 2
    return d


def rows_image(cxcywh, cls, score, nc=NC):
    """Decoded det_preds rows [n, 5 + nc]: obj = score, a one-hot class score of 1 (so score = obj exactly)."""
    n = len(cxcywh)
    d = np.zeros((n, 5 + nc), F32)
    d[:, :4] = cxcywh
    d[:, 4] = score
    d[np.arange(n), 5 + np.asarray(cls)] = 1.0
    return d


FAR_BOX = np.array([[605.0, 600.0, 10.0, 79.0]], F32)   # xyxy (600, 560.5, 610, 639.5): sets the max coordinate in y


def planted_rows(rng, kind, thr=0.65, n_pairs=12):
    """Planted near-threshold pairs for one image, cxcywh with classes and descending scores (a before b):
    "fused" pairs decided differently by the fused and the unfused denominator, "offset" pairs decided differently with
    and without the coordinate trick's shift (class 5..20, max coordinate 639.5 from FAR_BOX), "exact" pairs with fp32
    IoU exactly float32(thr), plus two zero-area boxes.  -> (cxcywh, cls, score, pairs [(ia, ib)])."""
    pa, pb = P.near_threshold_pairs(rng, 400, thr)
    A_, B_ = P.xyxy(*pa.T), P.xyxy(*pb.T)
    fused = P.suppresses_cuda(P.iou_cuda_f32(A_, B_), thr)
    unfused = P.suppresses_cuda(P.iou_cpu_f32(A_, B_), thr)
    cls = rng.integers(5, NC, len(pa))
    off = (cls.astype(F32) * F32(F32(639.5) + F32(1))).astype(F32)
    shifted = P.suppresses_cuda(P.iou_cuda_f32((A_ + off[:, None]).astype(F32), (B_ + off[:, None]).astype(F32)), thr)
    exact = P.iou_cuda_f32(A_, B_) == F32(thr)
    pick = {"fused": np.nonzero(fused != unfused)[0], "offset": np.nonzero(shifted != fused)[0],
            "exact": np.nonzero(exact)[0]}[kind]
    assert len(pick) >= n_pairs // 2, (kind, len(pick))
    pick = rng.choice(pick, min(n_pairs, len(pick)), replace=False)
    boxes, classes = [], []
    for k in pick:
        boxes += [pa[k], pb[k]]
        classes += [cls[k], cls[k]]
    boxes.append(FAR_BOX[0])
    classes.append(0)
    boxes += [[300.0, 300.0, 0.0, 12.0], [300.0, 300.0, 0.0, 12.0]]   # zero-area, same class
    classes += [7, 7]
    m = len(boxes)
    score = (np.linspace(0.95, 0.35, m)).astype(F32)
    return np.array(boxes, F32), np.array(classes), score, [(2 * i, 2 * i + 1) for i in range(len(pick))]


def negative_rows():
    """All coordinates negative (max -10): under the coordinate trick class 1, shifted by -9, overlaps class 0 with
    IoU 0.75 and suppresses it."""
    b = np.array([[-95, -95, -10, -10], [-100, -100, -10, -10], [-99.5, -100, -10.5, -10], [-300, -300, -200, -200]], F32)
    return to_cxcywh(b), np.array([1, 0, 0, 2]), np.array([0.9, 0.8, 0.7, 0.6], F32)


# ---------------------------------------------------------------------------------------------------------------------
# GPU harness: one production call, every stage read from its workspace, the call repeated for bit-identity
# ---------------------------------------------------------------------------------------------------------------------
def run_post(dev, preds, nc, conf, thr, agnostic=False, hw=None, strides=None, max_out=None):
    from gdrnpp_bop2022_b200 import _lib
    from gdrnpp_bop2022_b200.yolox_post import postprocess_padded

    x = torch.as_tensor(preds, dtype=torch.float32).to(dev)
    B, A = x.shape[:2]
    ws = [None]
    res = []
    for _ in range(2):
        if ws[0] is not None:
            ws[0].fill_(0xA5)   # stale contents must not leak into a rerun
        dets, n_det = postprocess_padded(x, nc, conf, thr, agnostic, hw=hw, strides=strides, max_out=max_out, workspace=ws)
        st = stage_views(ws[0], B, A, _lib)
        torch.cuda.synchronize()
        out = {"dets": dets.cpu().numpy(), "n_det": n_det.cpu().numpy()}
        n = st["n_cand"].cpu().numpy()
        out["n_cand"] = n
        out["max_coord"] = st["max_coord"].cpu().numpy()
        cand, score, order = st["cand"].cpu().numpy(), st["score"].cpu().numpy(), st["order"].cpu().numpy()
        mask = st["mask"].cpu().numpy().view(np.uint64)
        out["cand"] = [cand[b, :n[b]] for b in range(B)]
        out["score"] = [score[b, :n[b]] for b in range(B)]
        out["order"] = [order[b, :n[b]] for b in range(B)]
        out["mask"] = [mask[b, :n[b], :(n[b] + 63) // 64] for b in range(B)]
        res.append(out)
    a, b = res
    for k in ("dets", "n_det", "n_cand", "max_coord"):
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    for k in ("cand", "score", "order"):
        for u, v in zip(a[k], b[k]):
            assert np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8)), k
    for bi, (u, v) in enumerate(zip(a["mask"], b["mask"])):
        w = written_words(len(u))
        assert np.array_equal(u[w], v[w]), ("mask", bi)
    return a


def stage_views(ws, B, A, _lib):
    import ctypes

    off = (ctypes.c_size_t * 6)()
    _lib.check(_lib.lib().yolox_postprocess_layout(B, A, off), "yolox_postprocess_layout")
    base = (-ws.data_ptr()) % 256
    words = (A + 63) // 64

    def view(k, count, dtype, shape):
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return ws[base + off[k]: base + off[k] + nbytes].view(dtype).view(shape)

    return {"cand": view(0, B * A * 7, torch.float32, (B, A, 7)), "score": view(1, B * A, torch.float32, (B, A)),
            "order": view(2, B * A, torch.int32, (B, A)), "n_cand": view(3, B, torch.int32, (B,)),
            "max_coord": view(4, B, torch.float32, (B,)), "mask": view(5, B * A * words, torch.int64, (B, A, words))}


def written_words(n):
    """Boolean [n, words] of the mask words the kernel writes: word jb of row i when jb >= i // 64."""
    words = (n + 63) // 64
    return np.arange(words)[None, :] >= (np.arange(n) // 64)[:, None]


def oracle_mask(sorted_boxes, sorted_cls, thr, path, max_coord=None):
    """The words [n, words] of one image's suppression masks on a path: "trick", "vanilla" or "agnostic"."""
    b = np.asarray(sorted_boxes, F32)
    if path == "trick":
        off = (np.asarray(sorted_cls, F32) * F32(F32(max_coord) + F32(1))).astype(F32)
        b = (b + off[:, None]).astype(F32)
    sup = P.suppress_matrix(b, thr, "cuda", sorted_cls if path == "vanilla" else None)
    return P.mask_words(sup)


def pad_images(images, nc=NC):
    """list of [n_i, 5 + nc] -> [B, max n, 5 + nc]; padding rows have obj 0 (filtered out at conf > 0)."""
    A = max(1, max(len(d) for d in images))
    out = np.zeros((len(images), A, 5 + nc), F32)
    for i, d in enumerate(images):
        out[i, :len(d)] = d
    return out


# ---------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------
def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(F32)).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["shipped", "odd", "tta"])
def test_decode(dev, layout):
    """(x + grid) * stride and cx -+ w / 2 bit-exact against the fp32 replica; w, h = exp(wh) * stride within expf's
    2 ulp of fp64, and equal to torch's CUDA exp; xyxy bit-exact against torch's own decode.  Measured on an H100
    80GB HBM3 (700 W power limit): at most 1.76 ulp, and both equalities hold."""
    hw, strides = {"shipped": (HW_SHIPPED, STRIDES), "odd": ([(15, 20), (2, 3)], [8, 16]), "tta": tta_levels()}[layout]
    A = sum(h * w for h, w in hw)
    if layout == "tta":
        assert A == 43428
    rng = np.random.default_rng(10)
    gx, gy, st = P.anchor_grid(hw, strides)
    raw = np.zeros((3, A, 6), F32)
    raw[:, :, 4:] = 1.0   # every anchor scores 1: all pass, ranked in anchor order; nms_thr 2 keeps all
    # image 0: random centres, wh = 0 -> w = h = stride exactly: the centre and the conversion in isolation
    raw[0, :, :2] = rng.uniform(-0.5, 1.5, (A, 2))
    # image 1: centres cancel the grid (cx = cy = 0), so x2 = w / 2 exactly: w, h read back without rounding
    raw[1, :, 0], raw[1, :, 1] = -gx, -gy
    raw[1, :, 2:4] = rng.normal(0, 1.5, (A, 2))
    # image 2: everything random
    raw[2, :, :2] = rng.uniform(-0.5, 1.5, (A, 2))
    raw[2, :, 2:4] = rng.normal(0, 1.5, (A, 2))
    r = run_post(dev, raw, 1, 0.0, 2.0, True, hw=hw, strides=strides)
    assert r["n_cand"].tolist() == [A, A, A] and r["n_det"].tolist() == [A, A, A]
    for b in range(3):
        assert np.array_equal(r["order"][b], np.arange(A))
    cxcy, wh64 = P.decode(raw[0], hw, strides)
    want0 = P.xyxy(cxcy[:, 0], cxcy[:, 1], st.astype(F32), st.astype(F32))
    assert np.array_equal(r["cand"][0][:, :4], want0)
    # w, h: expf error, and equality with torch's CUDA exp
    w_k = (r["cand"][1][:, 2:4] * F32(2)).astype(F32)
    _, wh64 = P.decode(raw[1], hw, strides)
    err = np.abs(w_k.astype(np.float64) - wh64) / ulp32(wh64)
    t = torch.from_numpy(raw[1, :, 2:4]).to(dev)
    w_t = (torch.exp(t) * torch.from_numpy(st.astype(F32)).to(dev)[:, None]).cpu().numpy()
    print(f"decode {layout}: w/h max error {err.max():.3f} ulp, equal to torch's CUDA exp: {np.array_equal(w_k, w_t)}")
    assert err.max() <= 2.0
    # image 2 against the reference's decode + conversion on CUDA (torch ops, yolo_head.py / boxes.py)
    x = torch.from_numpy(raw[2]).to(dev)
    g = torch.from_numpy(np.stack([gx, gy], 1).astype(F32)).to(dev)
    s = torch.from_numpy(st.astype(F32)).to(dev)[:, None]
    xy, wh = (x[:, :2] + g) * s, torch.exp(x[:, 2:4]) * s
    ref = torch.cat([xy - wh / 2, xy + wh / 2], 1).cpu().numpy()
    assert np.array_equal(w_k, w_t)   # the kernel's expf is torch's CUDA exp, bit for bit
    assert np.array_equal(r["cand"][2][:, :4], ref)


# ---------------------------------------------------------------------------------------------------------------------
# filter and compaction
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_filter_and_compaction(dev):
    """Exact keep set, count and order: scores at float32(conf) and one ulp either side, score 0 at conf 0, class-score
    ties (the first maximum), every anchor passing, none passing, and random products whose rounding decides."""
    rng = np.random.default_rng(11)
    nc, A, conf = 5, 3000, 0.3
    d = random_dec(rng, A, nc)
    c32 = F32(conf)
    edge = np.array([np.nextafter(c32, F32(0)), c32, np.nextafter(c32, F32(1))], F32)
    for k, v in enumerate(np.tile(edge, 20)):
        d[40 * k, 4], d[40 * k, 5:] = 1.0, 0.0
        d[40 * k, 5 + k % nc] = v
    d[7::50, 5:] = 0.5   # every class score tied: class 0 wins
    d[9::50, 5:] = 0.0
    d[9::50, 5 + 3] = d[9::50, 5 + 4] = 0.6
    # products close to conf, where fp32 rounding of obj * cls decides
    near = rng.choice(np.nonzero(np.arange(A) % 10 == 3)[0], 250, replace=False)
    d[near, 4] = rng.uniform(0.4, 1, len(near)).astype(F32)
    d[near, 5:] = 0
    d[near, 5] = (conf / d[near, 4].astype(np.float64) * (1 + rng.normal(0, 3e-7, len(near)))).astype(F32)
    allpass = random_dec(rng, A, nc)
    nonepass = random_dec(rng, A, nc)
    nonepass[:, 4] = 0.01
    zero = random_dec(rng, A, nc)
    zero[::3, 4] = 0.0
    images = [(d, conf), (allpass, 0.0), (nonepass, 0.5), (zero, 0.0)]
    band = 0
    for img, cf in images:
        r = run_post(dev, img[None], nc, cf, 0.65)
        cc, cp = P.class_max(img[:, 5:])
        s32, keep, keep64 = P.score_filter(img[:, 4], cc, cf)
        cand = P.compact(keep)
        band += int((keep != keep64).sum())
        assert r["n_cand"][0] == len(cand)
        boxes = P.xyxy(*img[:, :4].T)
        want = np.concatenate([boxes, img[:, 4:5], cc[:, None], cp[:, None].astype(F32)], 1)[cand]
        assert np.array_equal(r["cand"][0], want)
        assert np.array_equal(r["score"][0], s32[cand])
        if len(cand):
            assert r["max_coord"][0] == boxes[cand].max()
    assert band > 0   # the near products include ones where fp32 rounding (not fp64) decides
    assert P.class_max(d[7:8, 5:])[1][0] == 0


# ---------------------------------------------------------------------------------------------------------------------
# rank
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rank(dev):
    """The exact permutation with heavily tied scores (8 levels), n = 1 .. 43 428 in one batch."""
    sizes = [1, 255, 256, 257, 1024, 1025, 8400, 43428]
    rng = np.random.default_rng(12)
    images = []
    for n in sizes:
        d = np.zeros((n, 6), F32)
        d[:, 0:2] = rng.uniform(0, 600, (n, 2))
        d[:, 2:4] = 0.0   # zero-area boxes: the NMS keeps all, so the ranking is the whole output order
        d[:, 4] = (rng.integers(1, 9, n) / 8).astype(F32)
        d[:, 5] = 1.0
        images.append(d)
    r = run_post(dev, pad_images(images, 1), 1, 0.01, 0.5, True)
    for b, n in enumerate(sizes):
        assert r["n_cand"][b] == n
        want = P.rank(images[b][:, 4])
        assert np.array_equal(r["order"][b], want), n
        assert r["n_det"][b] == n


# ---------------------------------------------------------------------------------------------------------------------
# mask
# ---------------------------------------------------------------------------------------------------------------------
def fp64_decisions(sorted_boxes, sorted_cls, path, max_coord):
    """(iou64 [n, n], band [n, n]): the IoU of every sorted pair in fp64 -- on the coordinate trick's boxes shifted in
    fp64 -- and the band around it within which the fp32 arithmetic may decide otherwise: 16 ulp of 1 for the IoU
    arithmetic, plus, on the trick path, 8 ulp of the largest shifted coordinate over the pair's shortest side."""
    b = np.asarray(sorted_boxes, np.float64)
    band = np.full((len(b), len(b)), 16 * 2.0 ** -24)
    if path == "trick":
        b = b + (np.asarray(sorted_cls, np.float64) * (float(max_coord) + 1))[:, None]
        big = np.abs(b).max(1)
        side = np.minimum(b[:, 2] - b[:, 0], b[:, 3] - b[:, 1])
        with np.errstate(divide="ignore"):
            band = band + 8 * np.spacing(np.maximum(big[:, None], big[None, :]).astype(F32)).astype(np.float64) / \
                np.minimum(side[:, None], side[None, :])
    return P.iou64(b[:, None, :], b[None, :, :]), band


@pytest.mark.gpu
@pytest.mark.parametrize("n", [63, 64, 65, 127, 128, 129])
def test_mask_words(dev, n):
    """Every mask word the kernel writes equals the oracle's bits: class-aware (coordinate trick: n <= 25 000) and
    class-agnostic images with planted fused-vs-unfused and offset-vs-unshifted pairs, IoU exactly at the threshold,
    zero-area boxes and negative-coordinate cross-class pairs; the per-class path in test_mask_words_vanilla.  Every
    pair whose fp64 IoU lies beyond the fp32 band is decided as in fp64."""
    rng = np.random.default_rng(100 + n)
    thr = 0.65
    images, planted, checked = [], [], 0
    for kind, agnostic in (("fused", True), ("offset", False), ("exact", False), ("exact", True), ("fused", False)):
        boxes_c, cls, score, pairs = planted_rows(rng, kind, thr, n_pairs=min(12, (n - 3) // 2 - 1))
        fill = n - len(boxes_c)
        fb = cluster_boxes(rng, fill)
        boxes_c = np.concatenate([boxes_c, to_cxcywh(fb)])
        cls = np.concatenate([cls, rng.integers(5, 9, fill)])
        score = np.concatenate([score, rng.uniform(0.05, 0.3, fill).astype(F32)])
        images.append((rows_image(boxes_c, cls, score), agnostic, pairs))
    nb, ncls, nscore = negative_rows()
    fill = n - 4
    neg_c = np.concatenate([nb, to_cxcywh(cluster_boxes(rng, fill) - F32(700))])
    images.append((rows_image(neg_c, np.concatenate([ncls, rng.integers(0, 3, fill)]),
                              np.concatenate([nscore, rng.uniform(0.05, 0.5, fill).astype(F32)])), False, []))
    for agnostic in (False, True):
        sel = [i for i, im in enumerate(images) if im[1] == agnostic]
        batch = pad_images([images[i][0] for i in sel])
        r = run_post(dev, batch, NC, 0.01, thr, agnostic)
        for b, i in enumerate(sel):
            dec, _, pairs = images[i]
            o = P.postprocess(dec, NC, 0.01, thr, agnostic)
            assert r["n_cand"][b] == n and np.array_equal(r["order"][b], o["order"])
            boxes = o["boxes"][o["cand"]][o["order"]]
            cls = np.argmax(dec[:, 5:], 1)[o["cand"]][o["order"]].astype(F32)
            path = "agnostic" if agnostic else "trick"
            want = oracle_mask(boxes, cls, thr, path, r["max_coord"][b])
            assert r["max_coord"][b] == o["boxes"][o["cand"]].max()
            got = r["mask"][b]
            w = written_words(n)
            diff = np.nonzero((got != want) & w)
            assert len(diff[0]) == 0, (path, i, diff)
            # outside the fp32 band every decision is the fp64 one
            bits = ((got[:, :, None] >> np.arange(64, dtype=np.uint64)) & np.uint64(1)).astype(bool).reshape(n, -1)[:, :n]
            i64, band = fp64_decisions(boxes, cls, path, r["max_coord"][b])
            beyond = np.triu(np.ones((n, n), bool), 1) & (np.abs(i64 - thr) > band)
            assert np.array_equal(bits[beyond], (i64 > thr)[beyond]), (path, i)
            checked += int(beyond.sum())
            inv = np.argsort(o["order"])   # candidate -> sorted position
            for ia, ib in pairs:
                lo, hi = sorted((inv[ia], inv[ib]))
                planted.append((i64[lo, hi], band[lo, hi]))
            # the greedy reduce over the kernel's own masks, and end to end
            kept = P.greedy_words(got, n)
            assert r["n_det"][b] == len(kept)
            assert np.array_equal(r["dets"][b, :len(kept)], o["rows"])
            assert np.array_equal(o["order"][kept], o["kept"])
    neg = images[-1][0]
    o = P.postprocess(neg, NC, 0.01, thr, False)
    assert 0 in o["kept"] and 1 not in o["kept"]   # class 1 at (-95, -95, -10, -10) suppressed class 0 through the shift
    dist = np.array([abs(i - thr) for i, _ in planted])
    inside = sum(abs(i - thr) <= band for i, band in planted)
    print(f"n={n}: {len(planted)} planted pairs, |iou64 - thr| from {dist.min():.2e} to {dist.max():.2e}, {inside} of them "
          f"inside the fp32 band; {checked} pairs beyond the band decided as in fp64")


@pytest.mark.gpu
def test_mask_words_vanilla(dev):
    """The class-aware path above 25 000 candidates (per class, unshifted): the mask words of the first 130 and the last
    70 sorted rows against the oracle, with planted fused-vs-unfused pairs at the top ranks."""
    rng = np.random.default_rng(19)
    thr, n = 0.65, 25001
    boxes_c, cls, score, _ = planted_rows(rng, "fused", thr, n_pairs=30)
    fill = n - len(boxes_c)
    boxes_c = np.concatenate([boxes_c, to_cxcywh(cluster_boxes(rng, fill, k=300))])
    cls = np.concatenate([cls, rng.integers(0, 4, fill)])
    score = np.concatenate([score, rng.uniform(0.02, 0.3, fill).astype(F32)])
    dec = rows_image(boxes_c, cls, score)
    r = run_post(dev, dec[None], NC, 0.01, thr, False)
    order = P.rank(score)
    assert r["n_cand"][0] == n and np.array_equal(r["order"][0], order)
    b, c = P.xyxy(*boxes_c.T)[order], cls[order]
    words = (n + 63) // 64
    for i in list(range(130)) + list(range(n - 70, n)):
        sup = np.zeros(words * 64, bool)
        sup[i + 1:n] = P.suppresses_cuda(P.iou_cuda_f32(b[i][None], b[i + 1:]), thr) & (c[i + 1:] == c[i])
        want = np.bitwise_or.reduce(sup.reshape(words, 64).astype(np.uint64) << np.arange(64, dtype=np.uint64), axis=1)
        jb = np.arange(words) >= i // 64
        assert np.array_equal(r["mask"][0][i][jb], want[jb]), i


# ---------------------------------------------------------------------------------------------------------------------
# reduce
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_reduce_cap_and_batch(dev):
    """The kept list against the oracle's greedy pass over the kernel's own masks and end to end, with max_out 1, 4,
    n - 1, n and A, over 4 images with different n, one of them empty."""
    rng = np.random.default_rng(13)
    sizes = [300, 0, 77, 1000]
    A = 1200
    images = []
    for n in sizes:
        b = cluster_boxes(rng, n, k=10)
        images.append(rows_image(to_cxcywh(b), rng.integers(0, 4, n), rng.uniform(0.05, 1, n).astype(F32)))
    batch = pad_images(images)
    batch = np.concatenate([batch, np.zeros((4, A - batch.shape[1], 5 + NC), F32)], 1)
    for agnostic in (False, True):
        o = [P.postprocess(d, NC, 0.01, 0.45, agnostic) if len(d) else None for d in images]
        nk = [len(x["kept"]) if x is not None else 0 for x in o]
        for max_out in sorted({1, 4, max(nk) - 1, max(nk), A}):
            r = run_post(dev, batch, NC, 0.01, 0.45, agnostic, max_out=max_out)
            for b, n in enumerate(sizes):
                assert r["n_cand"][b] == n
                if n == 0:
                    assert r["n_det"][b] == 0
                    continue
                kept = P.greedy_words(r["mask"][b], n, max_out)
                assert r["n_det"][b] == min(nk[b], max_out) == len(kept)
                assert np.array_equal(r["dets"][b, :len(kept)], o[b]["rows"][:max_out])
                assert not r["dets"][b, len(kept):].any()


@pytest.mark.gpu
def test_anchor_limit(dev):
    from gdrnpp_bop2022_b200._lib import GdrnError
    from gdrnpp_bop2022_b200.yolox_post import postprocess_padded

    for A, ok in ((65536, True), (65537, False)):
        x = torch.zeros((1, A, 6), device=dev)
        x[0, :5, :4] = torch.tensor([10.0, 10.0, 4.0, 4.0], device=dev)
        x[0, :5, 4:] = 1.0
        if ok:
            dets, n = postprocess_padded(x, 1, 0.5, 0.5, max_out=8)
            assert int(n[0]) == 1
        else:
            with pytest.raises(GdrnError, match="65536"):
                postprocess_padded(x, 1, 0.5, 0.5, max_out=8)
        del x
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# against torchvision on the GPU
# ---------------------------------------------------------------------------------------------------------------------
def ref_postprocess(dec, nc, conf, thr, agnostic):
    """det/yolox/utils/boxes.py:34-80 on one image of decoded det_preds (CUDA tensors), with torchvision's ops."""
    import torchvision

    p = dec.clone()
    box = torch.stack([p[:, 0] - p[:, 2] / 2, p[:, 1] - p[:, 3] / 2, p[:, 0] + p[:, 2] / 2, p[:, 1] + p[:, 3] / 2], 1)
    p[:, :4] = box
    cc, cp = torch.max(p[:, 5:5 + nc], 1, keepdim=True)
    m = (p[:, 4] * cc.squeeze() >= conf).squeeze()
    det = torch.cat((p[:, :5], cc, cp.float()), 1)[m]
    if not det.size(0):
        return det
    if agnostic:
        keep = torchvision.ops.nms(det[:, :4], det[:, 4] * det[:, 5], thr)
    else:
        keep = torchvision.ops.batched_nms(det[:, :4], det[:, 4] * det[:, 5], det[:, 6], thr)
    return det[keep]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [20, 100, 3000, 43428])
def test_torch_cuda_sort_tie_order(dev, n):
    """Measures whether torch's CUDA sort (and torchvision's CUDA nms, which sorts internally) keep tied scores in index
    order, at n <= 32, <= 128, <= 4096 and above.  On an H100 80GB HBM3 with torch 2.11 and torchvision 0.26,
    torch.sort(descending=True) did not at n <= 32 and did above; nms did at every size, and that is asserted: the
    coordinate-trick and agnostic comparisons below may have ties.  The per-class path ends with torch.sort, so the
    comparisons that reach it use distinct scores by construction."""
    import torchvision

    g = torch.Generator().manual_seed(n)
    s = (torch.randint(0, 8, (n,), generator=g).float() / 8).to(dev)
    stable = P.rank(s.cpu().numpy())
    default = torch.sort(s, descending=True)[1].cpu().numpy()
    ar = torch.arange(n, device=dev, dtype=torch.float32) * 10
    bx = torch.stack([ar, torch.zeros_like(ar), ar + 5, torch.full_like(ar, 5.0)], 1)
    nms_order = torchvision.ops.nms(bx, s, 0.5).cpu().numpy()
    print(f"n={n}: torch.sort(descending) keeps ties in index order: {np.array_equal(default, stable)}; "
          f"torchvision nms: {np.array_equal(nms_order, stable)}")
    assert np.array_equal(nms_order, stable)   # torchvision's nms sorts stably: the rank kernel's order


@pytest.mark.gpu
@pytest.mark.parametrize("agnostic", [False, True])
def test_vs_torchvision_planted(dev, agnostic):
    """Kept rows and their order equal torchvision's batched_nms / nms on CUDA, fed the reference's decode, on images of
    planted near-threshold pairs (fused, offset, exact; one image with tied scores) and negative-coordinate cross-class
    pairs."""
    rng = np.random.default_rng(14)
    thr = 0.65
    images = []
    for kind in ("fused", "offset", "exact"):
        for _ in range(3):
            boxes_c, cls, score, _ = planted_rows(rng, kind, thr, n_pairs=16)
            images.append(rows_image(boxes_c, cls, score))
    boxes_c, cls, score, _ = planted_rows(rng, "fused", thr, n_pairs=16)
    images.append(rows_image(boxes_c, cls, (np.ceil(score * 4) / 4).astype(F32)))   # tied scores: nms sorts stably
    nb, ncls, nscore = negative_rows()
    images.append(rows_image(nb, ncls, nscore))
    batch = pad_images(images)
    r = run_post(dev, batch, NC, 0.01, thr, agnostic)
    x = torch.from_numpy(batch).to(dev)
    for b in range(len(images)):
        ref = ref_postprocess(x[b], NC, 0.01, thr, agnostic).cpu().numpy()
        assert r["n_det"][b] == len(ref), b
        assert np.array_equal(r["dets"][b, :len(ref)], ref), b


@pytest.mark.gpu
@pytest.mark.parametrize("n", [25000, 25001])
def test_vs_torchvision_trick_cutoff(dev, n):
    """Both sides of batched_nms' switch from the coordinate trick to the per-class path: near-threshold pairs whose
    decision the offsets change, among n candidates of 21 classes (distinct scores)."""
    rng = np.random.default_rng(15 + n)
    thr = 0.65
    boxes_c, cls, _, pairs = planted_rows(rng, "offset", thr, n_pairs=40)
    fill = n - len(boxes_c)
    fb = cluster_boxes(rng, fill, k=400)
    boxes_c = np.concatenate([boxes_c, to_cxcywh(fb)])
    cls = np.concatenate([cls, rng.integers(0, NC, fill)])
    score = (1 - np.arange(n) / (2 * n)).astype(F32)   # distinct, planted pairs first
    dec = rows_image(boxes_c, cls, score)
    r = run_post(dev, dec[None], NC, 0.01, thr, False)
    ref = ref_postprocess(torch.from_numpy(dec).to(dev), NC, 0.01, thr, False).cpu().numpy()
    assert r["n_cand"][0] == n
    assert r["n_det"][0] == len(ref)
    assert np.array_equal(r["dets"][0, :len(ref)], ref)
    # the planted rows rank above every filler row, so their fate is decided among themselves: on both sides of the
    # switch the two paths disagree about them, so the comparison above pins the cutoff
    top = len(pairs) * 2 + 3
    pb_ = P.xyxy(*boxes_c[:top].T)
    off = (cls[:top].astype(F32) * F32(P.xyxy(*boxes_c.T).max() + F32(1))).astype(F32)
    trick = P.greedy(P.suppress_matrix((pb_ + off[:, None]).astype(F32), thr, "cuda"))
    vanilla = P.greedy(P.suppress_matrix(pb_, thr, "cuda", cls[:top]))
    assert not np.array_equal(trick, vanilla)
    want = trick if n <= P.TRICK_MAX_CANDIDATES else vanilla
    got = np.nonzero(np.isin(score[:top], r["dets"][0, :r["n_det"][0], 4]))[0]
    assert np.array_equal(got, want)


@pytest.mark.gpu
def test_vs_torchvision_shipped_tta(dev):
    """The shipped settings: 21 classes, conf 0.001, nms 0.65, the TTA anchor count 43 428 (every anchor passes, so
    torchvision takes the per-class path); distinct scores."""
    rng = np.random.default_rng(16)
    A = 43428
    dec = np.zeros((2, A, 5 + NC), F32)
    for b in range(2):
        fb = cluster_boxes(rng, A, k=60)
        dec[b, :, :4] = to_cxcywh(fb)
        dec[b, :, 4] = (1 - rng.permutation(A) / (2 * A)).astype(F32)
        dec[b, :, 5:] = rng.uniform(0.002, 0.5, (A, NC)).astype(F32)
        dec[b, np.arange(A), 5 + rng.integers(0, NC, A)] = 1.0
    r = run_post(dev, dec, NC, 0.001, 0.65, False)
    x = torch.from_numpy(dec).to(dev)
    for b in range(2):
        assert r["n_cand"][b] == A
        ref = ref_postprocess(x[b], NC, 0.001, 0.65, False).cpu().numpy()
        assert r["n_det"][b] == len(ref)
        assert np.array_equal(r["dets"][b, :len(ref)], ref)


# ---------------------------------------------------------------------------------------------------------------------
# keep-single-instance (csrc/yolox_net.cu)
# ---------------------------------------------------------------------------------------------------------------------
def run_ksi(dev, preds, nc, conf, thr):
    import ctypes

    from gdrnpp_bop2022_b200 import _lib
    from gdrnpp_bop2022_b200.predictor_yolo import postprocess_single_instance

    x = torch.as_tensor(preds, dtype=torch.float32).to(dev)
    B, A = x.shape[:2]
    off = (ctypes.c_size_t * 3)()
    _lib.check(_lib.lib().yolox_postprocess_single_layout(B, A, nc, off), "yolox_postprocess_single_layout")
    ws = [None]
    res = []
    for _ in range(2):
        dets, n = postprocess_single_instance(x, nc, conf, thr, workspace=ws)
        base = (-ws[0].data_ptr()) % 256
        sel = ws[0][base + off[2]: base + off[2] + B * nc * 4].view(torch.int32).view(B, nc)
        score = ws[0][base + off[0]: base + off[0] + B * A * 4].view(torch.float32).view(B, A)
        res.append((dets.cpu().numpy(), n.cpu().numpy(), sel.cpu().numpy(), score.cpu().numpy()))
    for u, v in zip(*res):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    return res[0]


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [1, 21, 1024])
def test_ksi_selection(dev, nc):
    """Per class the anchor the reference's loop picks: equal scores -> the lowest anchor, a score of exactly conf
    passes, a score of 0 never counts; rows in ascending class order."""
    rng = np.random.default_rng(17 + nc)
    A, conf = 3000, 0.3
    images = []
    for b in range(3):
        d = random_dec(rng, A, nc)
        d[:, 4] = (rng.integers(1, 9, A) / 8).astype(F32)   # heavy ties of scores and of class scores
        d[:, 5:] = (rng.integers(0, 9, (A, nc)) / 8).astype(F32)
        if b == 1:
            d[:, 4] = 1.0
            d[:, 5:] = 0.0
            d[np.arange(A), 5 + rng.integers(0, nc, A)] = F32(conf)   # every score exactly float32(conf)
        if b == 2:
            d[:, 4] = 0.0   # nothing
        images.append(d)
    batch = np.stack(images)
    dets, n, sel, score = run_ksi(dev, batch, nc, conf, 0.65)
    for b, d in enumerate(images):
        cc, cp = P.class_max(d[:, 5:])
        s32, keep, _ = P.score_filter(d[:, 4], cc, conf)
        assert np.array_equal(score[b], s32)
        want_sel = P.ksi_select(s32, cp, keep, nc)
        assert np.array_equal(sel[b], want_sel), b
        _, rows = P.keep_single_instance(d, nc, conf, 0.65)
        assert n[b] == len(rows)
        assert np.array_equal(dets[b, :n[b]], rows)
        assert (np.diff(dets[b, :n[b], 6]) > 0).all()
    assert n[1] > 0 and n[2] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("thr", [0.65, 0.3, 0.6])
def test_ksi_nms_vs_torchvision_cpu(dev, thr):
    """Keep-single-instance NMS against torchvision's CPU nms on the same rows (what the reference runs), with pairs
    near the threshold, including fp32 IoUs equal to float32(thr)."""
    import torchvision

    rng = np.random.default_rng(18)
    pa, pb = P.near_threshold_pairs(rng, 600, thr, span=24)
    A_, B_ = P.xyxy(*pa.T), P.xyxy(*pb.T)
    i32 = P.iou_cpu_f32(A_, B_)
    flips = np.nonzero(P.suppresses_cpu(i32, thr) != (i32 > F32(thr)))[0]
    if F32(thr) > thr:
        assert len(flips) > 0   # the threshold rounds up: equal fp32 IoUs are the float / double difference
    idx = np.concatenate([flips[:60], rng.choice(len(pa), 120, replace=False)])
    m = len(idx)
    nc = 3
    d = np.zeros((m, 3, 5 + nc), F32)
    d[:, 0, :4], d[:, 1, :4] = pa[idx], pb[idx]
    d[:, 2, :4] = [900, 900, 10, 10]
    d[:, :, 4] = [0.9, 0.8, 0.7]
    d[:, 0, 5], d[:, 1, 6], d[:, 2, 7] = 1.0, 1.0, 1.0
    dets, n, _, _ = run_ksi(dev, d, nc, 0.01, thr)
    for k in range(m):
        _, rows = P.keep_single_instance(d[k], nc, 0.01, thr)
        bx = torch.from_numpy(P.xyxy(*d[k, :, :4].T))
        keep = torchvision.ops.nms(bx, torch.from_numpy(d[k, :, 4].copy()), thr).numpy()
        ref = rows[np.argsort(rows[:, 6])]
        assert sorted(keep.tolist()) == ref[:, 6].astype(int).tolist()
        assert n[k] == len(ref) and np.array_equal(dets[k, :n[k]], ref), (k, thr)


@pytest.mark.gpu
def test_ksi_class_limit(dev):
    from gdrnpp_bop2022_b200._lib import GdrnError
    from gdrnpp_bop2022_b200.predictor_yolo import postprocess_single_instance

    x = torch.zeros((1, 4, 5 + 1025), device=dev)
    with pytest.raises(GdrnError, match="problem size"):
        postprocess_single_instance(x, 1025, 0.3, 0.65)
