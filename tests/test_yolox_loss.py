"""The YOLOX training loss (gdrnpp_bop2022_b200/yolox_loss.py, csrc/yolox_loss.cu) against the reference's own
get_losses (tests/golden/ref_yolox_loss.npz, made by tools/make_golden_ref_yolox_loss.py) and the torch restatement in
oracle/yolox_loss_oracle.py.

CPU: the fp64 oracle reproduces the golden assignment, losses and gradients.  GPU: every kernel stage on the kernel's
own input to it (candidates bit-exact with the fp32 replica, IoU and cost against fp64, k, the per-GT choice and the
conflict resolution exactly), then losses and gradients against fp64 autograd through the oracle, end to end against
the golden file, fp16 inputs, a real YoloxTrainBatcher batch and a conv whose weights are leaves.  Every GPU call runs
twice and must give bit-identical results.

The assignment is compared exactly where the reference's recorded decision margins exceed 1e-5 (a GT's k-th and
(k+1)-th cost, and its top-10 IoU sum against an integer); every golden case has all its margins above that.
"""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import yolox_loss_oracle as O

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_yolox_loss.npz")
MARGIN = 1e-5
# the reference's fp32 IoU: box edges near 800 px cancel in br - tl, up to ~2e-6 off for small overlaps
IOU_REF_ATOL = 5e-6
KEYS = ("loss_iou", "loss_conf", "loss_cls", "loss_l1")


def head(C, use_l1, iou="iou", cls="bce", obj="bce"):
    return SimpleNamespace(num_classes=C, use_l1=use_l1, iou_loss=SimpleNamespace(loss_type=iou), cls_loss_type=cls,
                           obj_loss_type=obj)


def inputs(case, dtype=torch.float64, device="cpu"):
    """(x_shifts, y_shifts, expanded_strides, labels, outputs leaf, origin leaf) of a case in ``dtype``."""
    seed, B, side, C, n_gts, kind, use_l1 = case
    xs, ys, es, labels, raw = O.make_case(seed, B, side, C, n_gts, kind)
    cv = lambda t: t.to(dtype=dtype, device=device)  # noqa: E731
    xs, ys, es = [cv(t) for t in xs], [cv(t) for t in ys], [cv(t) for t in es]
    outputs = O.decode(raw.double(), [t.double() for t in xs], [t.double() for t in ys], [t.double() for t in es])
    outputs = cv(outputs.float()).requires_grad_(True)
    origin = cv(raw[..., :4]).requires_grad_(True)
    return xs, ys, es, cv(labels), outputs, origin


def levels(origin, xs):
    return list(torch.split(origin, [x.shape[1] for x in xs], 1))


def total(losses):
    return sum(w * losses[k] for k, w in O.LOSS_WEIGHTS.items() if torch.is_tensor(losses[k]))


def rel_err(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want).max() / max(np.abs(want).max(), 1e-30) if want.size else 0.0


def golden(name):
    z = np.load(GOLDEN)
    return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}


def assert_matches_golden(name, fg, matched, iou_t, losses, g_out, g_org, iou_atol):
    """fg [B, A] bool, matched [B, A], iou_t [B, A], losses (4 floats), gradients dense as numpy."""
    ref = golden(name)
    assert (ref["margins"] > MARGIN).all(), "a golden case with a margin at the tie threshold"
    want_fg = np.zeros_like(fg)
    want_fg[tuple(ref["fg_idx"].T)] = True
    np.testing.assert_array_equal(fg, want_fg)
    np.testing.assert_array_equal(matched[fg], ref["matched"])
    np.testing.assert_allclose(iou_t[fg], ref["iou_t"], rtol=0, atol=iou_atol)
    np.testing.assert_allclose(losses, ref["losses"], rtol=1e-5, atol=0)
    assert rel_err(g_out[..., 4], ref["grad_obj"]) < 1e-5
    rows = np.zeros(fg.shape, bool)
    rows[tuple(ref["grad_rows"].T)] = True
    np.testing.assert_array_equal(rows, fg)
    assert rel_err(g_out[rows], ref["grad_out_rows"]) < 1e-5
    off = g_out.copy()
    off[rows] = 0
    off[..., 4] = 0
    assert not off.any()
    orows = np.zeros(fg.shape, bool)
    if len(ref["grad_origin_rows_idx"]):
        orows[tuple(ref["grad_origin_rows_idx"].T)] = True
    assert rel_err(g_org[orows], ref["grad_origin_rows"]) < 1e-5
    assert not g_org[~orows].any()


# --------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", list(O.GOLDEN_CASES))
def test_oracle_reproduces_reference(name):
    case = O.GOLDEN_CASES[name]
    C, use_l1 = case[3], case[6]
    xs, ys, es, labels, outputs, origin = inputs(case)
    trace = []
    out, losses = O.get_losses(head(C, use_l1), None, xs, ys, es, labels, outputs, levels(origin, xs), torch.float64,
                               trace=trace)
    total(losses).backward()
    B, A = outputs.shape[:2]
    fg = np.zeros((B, A), bool)
    matched = np.full((B, A), -1)
    iou_t = np.zeros((B, A))
    for b, r in enumerate(trace):
        if r is not None:
            fg[b], matched[b], iou_t[b] = r["fg"].numpy(), r["matched"].numpy(), r["iou_t"].numpy()
    got = [float(losses[k].detach()) if torch.is_tensor(losses[k]) else losses[k] for k in KEYS]
    g_org = origin.grad.numpy() if origin.grad is not None else np.zeros(origin.shape)
    assert_matches_golden(name, fg, matched, iou_t, got, outputs.grad.numpy(), g_org, iou_atol=IOU_REF_ATOL)
    assert (losses["loss_l1"] == 0.0) == (not use_l1)


def test_oracle_gt_without_candidate_takes_nothing():
    xs, ys, es, labels, raw = O.make_case(9, 2, 448, 30, (4, 6), "nocand")
    outputs = O.decode(raw.double(), [t.double() for t in xs], [t.double() for t in ys], [t.double() for t in es])
    trace = []
    _, losses = O.get_losses(head(30, True), None, [t.double() for t in xs], [t.double() for t in ys],
                             [t.double() for t in es], labels.double(), outputs, levels(raw[..., :4].double(), xs),
                             torch.float64, trace=trace)
    assert all(not r["fg"].any() and not r["cand"].any() for r in trace)
    assert float(losses["loss_iou"]) == 0 and float(losses["loss_cls"]) == 0 and float(losses["loss_conf"]) > 0


@pytest.mark.parametrize("opt, value", [("iou", "giou"), ("cls", "focal"), ("obj", "focal")])
def test_rejects_unsupported_options(opt, value):
    from gdrnpp_bop2022_b200 import yolox_loss as Y

    name = {"iou": "iou_loss_type", "cls": "cls_loss_type", "obj": "obj_loss_type"}[opt]
    with pytest.raises(NotImplementedError, match=name):
        Y.get_losses(head(30, False, **{opt: value}), None, [], [], [], torch.zeros(1, 1, 5), torch.zeros(1, 1, 35), [],
                     torch.float32)


# --------------------------------------------------------------------------------------------------------- GPU
def kernel_stages(dev, xs, ys, es, labels, outputs, origin, C, use_l1):
    """One forward of the kernels with the pair trace; -> dict of numpy stage results.  Run twice: bit-identical."""
    from gdrnpp_bop2022_b200 import yolox_loss as Y

    B, A = outputs.shape[:2]
    M = labels.shape[1]
    out = outputs.detach().to(dev).contiguous()
    org = origin.detach().to(dev).to(out.dtype).contiguous() if use_l1 else None
    shifts = torch.cat(xs + ys + es, 1).to(dev, torch.float32).reshape(3, -1)
    lab = labels.to(dev, torch.float32).contiguous()
    runs = []
    for _ in range(2):
        trace = torch.zeros(B, M, A, 3, device=dev)
        ws, offs = Y.forward_raw(out, org, lab, shifts, C, use_l1, trace)
        v = lambda n, dt, shape: Y.workspace_view(ws, offs, n, dt, shape).cpu().numpy()  # noqa: E731
        runs.append(dict(
            nlabel=v("nlabel", torch.int32, (B,)), cand=v("cand", torch.uint8, (B, A)).astype(bool),
            n_cand=v("n_cand", torch.int32, (B,)), k=v("k", torch.int32, (B, M)), iou_sum=v("iou_sum", torch.float32, (B, M)),
            chosen=v("chosen", torch.int32, (B, M, 10)), fg=v("fg", torch.uint8, (B, A)).astype(bool),
            matched=v("matched", torch.int32, (B, A)), iou_t=v("iou_t", torch.float32, (B, A)),
            result=v("result", torch.float32, (8,)), trace=trace.cpu().numpy()))
        torch.cuda.synchronize()
    for key in runs[0]:
        assert np.array_equal(runs[0][key], runs[1][key], equal_nan=True), key
    return runs[0]


def check_stages(st, xs, ys, es, labels, outputs, C):
    """Each stage against the oracle on the kernel's own input.  -> number of near-integer k skipped."""
    x = torch.cat(xs, 1)[0].float().cpu().numpy()
    y = torch.cat(ys, 1)[0].float().cpu().numpy()
    s = torch.cat(es, 1)[0].float().cpu().numpy()
    lab32 = labels.float().cpu()
    o64 = outputs.detach().double().cpu()
    nl = O.num_labels(lab32)
    np.testing.assert_array_equal(st["nlabel"], nl)
    skipped = 0
    for b, n in enumerate(nl):
        if n == 0:
            assert not st["cand"][b].any() and not st["fg"][b].any()
            continue
        gt32 = lab32[b, :n, 1:5].numpy()
        cand, both = O.replay_candidates(gt32, x, y, s)
        np.testing.assert_array_equal(st["cand"][b], cand)                     # bit-exact with the fp32 replica
        ci = np.nonzero(cand)[0]
        assert st["n_cand"][b] == len(ci)
        if len(ci) == 0:   # no candidate: the GTs take nothing
            assert not st["fg"][b].any() and (st["k"][b, :n] == 0).all()
            continue
        tr = st["trace"][b, :n][:, ci]
        iou_k, c0_k, cost_k = tr[..., 0], tr[..., 1], tr[..., 2]
        ious64, c064 = O.pair_costs(lab32[b, :n, 1:5].double(), lab32[b, :n, 0], o64[b, ci, :4], o64[b, ci, 4:5],
                                    o64[b, ci, 5:], C)
        assert np.abs(iou_k - ious64.numpy()).max() <= 1e-6
        np.testing.assert_allclose(c0_k, c064.numpy(), rtol=1e-5, atol=1e-6)
        bo = both[:, ci]
        np.testing.assert_array_equal(cost_k[bo], c0_k[bo])
        np.testing.assert_array_equal(cost_k[~bo], (c0_k[~bo] + np.float32(100000.0)).astype(np.float32))
        k_want, s64 = O.replay_k(iou_k)
        near = np.abs(s64 - np.round(s64)) < MARGIN
        skipped += int(near.sum())
        np.testing.assert_array_equal(st["k"][b, :n][~near], k_want[~near])
        np.testing.assert_allclose(st["iou_sum"][b, :n], s64, rtol=1e-5, atol=1e-6)
        chosen, fg_c, m_c = O.replay_choice(cost_k, st["k"][b, :n])
        for g in range(n):
            kk = st["k"][b, g]
            got = st["chosen"][b, g]
            assert (got[kk:] == -1).all()
            np.testing.assert_array_equal(np.sort(got[:kk]), ci[chosen[g]])
        fg = np.zeros(len(cand), bool)
        fg[ci] = fg_c
        np.testing.assert_array_equal(st["fg"][b], fg)
        np.testing.assert_array_equal(st["matched"][b][ci], m_c)
        assert (st["matched"][b][~fg] == -1).all()
        # the IoU target is the kernel's own pair IoU with the final GT
        fi = np.nonzero(fg_c)[0]
        np.testing.assert_array_equal(st["iou_t"][b][ci[fi]], iou_k[m_c[fi], fi])
    return skipped


def run_gpu_loss(dev, xs, ys, es, labels, outputs, origin, C, use_l1, upstream=None):
    """get_losses + backward on the GPU, twice, bit-identical.  -> (losses, ratio, grad outputs, grad origin) on CPU."""
    from gdrnpp_bop2022_b200 import yolox_loss as Y

    res = []
    for _ in range(2):
        out = outputs.detach().to(dev).requires_grad_(True)
        org = origin.detach().to(dev).requires_grad_(True)
        o, L = Y.get_losses(head(C, use_l1), None, [t.to(dev) for t in xs], [t.to(dev) for t in ys],
                            [t.to(dev) for t in es], labels.to(dev), out, levels(org, xs), out.dtype)
        tot = total(L) if upstream is None else sum(u * L[k] for k, u in zip(KEYS, upstream) if torch.is_tensor(L[k]))
        tot.backward()
        assert (L["loss_l1"] == 0.0) == (not use_l1) and o["num_fg"].dim() == 0 and o["num_fg"].is_cuda
        g_org = org.grad if org.grad is not None else torch.zeros_like(org)
        assert out.grad.dtype == outputs.dtype and g_org.dtype == origin.dtype
        res.append((torch.stack([L[k].detach() if torch.is_tensor(L[k]) else torch.zeros((), device=dev) for k in KEYS]),
                    o["num_fg"], out.grad, g_org))
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())
    return tuple(t.cpu() for t in res[0])


def oracle_on_assignment(st, xs, ys, es, labels, outputs, origin, C, use_l1, upstream=None):
    """fp64 autograd through the oracle's loss on the kernel's assignment.  -> (losses, grad outputs, grad origin)."""
    out = outputs.detach().double().cpu().requires_grad_(True)
    org = origin.detach().double().cpu().requires_grad_(True)
    cat = lambda ts: torch.cat(ts, 1)[0].double().cpu()  # noqa: E731
    fg = torch.from_numpy(st["fg"])
    matched = torch.from_numpy(st["matched"]).long().clamp(min=0)
    iou_t = torch.from_numpy(st["iou_t"]).double()
    li, lo, lc, ll, _ = O.losses_from_assignment(out, org if use_l1 else None, labels.double().cpu(), fg, matched, iou_t,
                                                 cat(xs), cat(ys), cat(es), C, use_l1)
    L = dict(zip(KEYS, (li, lo, lc, ll)))
    tot = total(L) if upstream is None else sum(u * L[k] for k, u in zip(KEYS, upstream) if torch.is_tensor(L[k]))
    tot.backward()
    g_org = org.grad if org.grad is not None else torch.zeros_like(org)
    return np.array([float(L[k].detach()) if torch.is_tensor(L[k]) else L[k] for k in KEYS]), out.grad.numpy(), g_org.numpy()


def check_case(dev, xs, ys, es, labels, outputs, origin, C, use_l1):
    st = kernel_stages(dev, xs, ys, es, labels, outputs, origin, C, use_l1)
    skipped = check_stages(st, xs, ys, es, labels, outputs, C)
    losses, ratio, g_out, g_org = run_gpu_loss(dev, xs, ys, es, labels, outputs, origin, C, use_l1)
    want, w_out, w_org = oracle_on_assignment(st, xs, ys, es, labels, outputs, origin, C, use_l1)
    np.testing.assert_allclose(losses.double().numpy(), want, rtol=1e-5, atol=0)
    assert rel_err(g_out.double().numpy(), w_out) < 1e-5
    assert rel_err(g_org.double().numpy(), w_org) < 1e-5 or not use_l1
    assert float(ratio) == pytest.approx(st["fg"].sum() / max(sum(O.num_labels(labels.float().cpu())), 1), rel=1e-6)
    return st, skipped


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["s640", "s640_nol1", "tiny", "dup", "border"])
def test_stages_losses_and_gradients(dev, name):
    case = O.GOLDEN_CASES[name]
    xs, ys, es, labels, outputs, origin = inputs(case, torch.float32)
    _, skipped = check_case(dev, xs, ys, es, labels, outputs, origin, case[3], case[6])
    assert skipped <= 2


@pytest.mark.gpu
def test_gt_without_candidate_takes_nothing(dev):
    xs, ys, es, labels, raw = O.make_case(9, 2, 448, 30, (4, 6), "nocand")
    labels[0, :3] = O.make_labels(torch.Generator().manual_seed(3), 1, 448, 30, (3,))[0, :3]   # image 0 has candidates
    outputs = O.decode(raw, xs, ys, es)
    st, _ = check_case(dev, xs, ys, es, labels, outputs, raw[..., :4], 30, True)
    assert st["fg"][0].any() and not st["fg"][1].any() and st["n_cand"][1] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(O.GOLDEN_CASES))
def test_end_to_end_matches_reference(dev, name):
    case = O.GOLDEN_CASES[name]
    xs, ys, es, labels, outputs, origin = inputs(case, torch.float32)
    st = kernel_stages(dev, xs, ys, es, labels, outputs, origin, case[3], case[6])
    losses, _, g_out, g_org = run_gpu_loss(dev, xs, ys, es, labels, outputs, origin, case[3], case[6])
    assert_matches_golden(name, st["fg"], st["matched"], st["iou_t"], losses.double().numpy(), g_out.numpy(),
                          g_org.numpy(), iou_atol=IOU_REF_ATOL)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_precision_inputs(dev, dtype):
    """AMP: fp16 (or bf16) outputs and labels; computed in fp32 on the values given, gradients in the input dtype."""
    case = O.GOLDEN_CASES["s640"]
    xs, ys, es, labels, outputs, origin = inputs(case, dtype)
    labels_h = labels
    st = kernel_stages(dev, xs, ys, es, labels_h, outputs, origin, 30, True)
    check_stages(st, xs, ys, es, labels_h, outputs, 30)
    losses, _, g_out, g_org = run_gpu_loss(dev, xs, ys, es, labels_h, outputs, origin, 30, True)
    want, w_out, w_org = oracle_on_assignment(st, xs, ys, es, labels_h, outputs, origin, 30, True)
    np.testing.assert_allclose(losses.double().numpy(), want, rtol=1e-5, atol=0)
    tol = 2e-3 if dtype == torch.float16 else 1e-2   # the gradient rounded to the input dtype
    assert rel_err(g_out.double().numpy(), w_out) < tol and rel_err(g_org.double().numpy(), w_org) < tol


@pytest.mark.gpu
def test_scaled_upstream_overflow(dev):
    """GradScaler's inf: every gradient the reference computes turns non-finite where the oracle's does, rows it never
    touches stay zero."""
    case = O.GOLDEN_CASES["s448"]
    xs, ys, es, labels, outputs, origin = inputs(case, torch.float32)
    up = (float("inf"), float("inf"), float("inf"), float("inf"))
    st = kernel_stages(dev, xs, ys, es, labels, outputs, origin, 30, True)
    _, _, g_out, g_org = run_gpu_loss(dev, xs, ys, es, labels, outputs, origin, 30, True, upstream=up)
    _, w_out, w_org = oracle_on_assignment(st, xs, ys, es, labels, outputs, origin, 30, True, upstream=up)
    g_out, g_org = g_out.numpy(), g_org.numpy()
    np.testing.assert_array_equal(np.isfinite(g_out[..., 4:]), np.isfinite(w_out[..., 4:]))
    np.testing.assert_array_equal(np.isfinite(g_org), np.isfinite(w_org))
    fg = st["fg"]
    assert not np.isfinite(g_out[fg][:, :4]).all(axis=1).any()
    assert (g_out[~fg][:, :4] == 0).all() and (g_out[~fg][:, 5:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [30.0, -1.0])
def test_class_id_out_of_range_is_rejected(dev, bad):
    xs, ys, es, labels, outputs, origin = inputs(O.GOLDEN_CASES["s448"], torch.float32)
    labels[1, 3, 0] = bad
    with pytest.raises(ValueError, match="class id"):
        run_gpu_loss(dev, xs, ys, es, labels, outputs, origin, 30, True)


@pytest.mark.gpu
def test_train_batcher_labels(dev, tmp_path):
    """labels of a real YoloxTrainBatcher batch of the synthetic LM-O split (640 x 640, up to 120 rows per image)."""
    from gdrnpp_bop2022_b200 import synthetic
    from gdrnpp_bop2022_b200 import yolox_train_batch as YT
    from gdrnpp_bop2022_b200.yolox_model import load_yolox_config

    synthetic.write_bop_train_tree(str(tmp_path), dataset="lmo", num_images=12, obj_ids=(1, 5, 6, 2), insts_per_image=4)
    cfg = load_yolox_config(synthetic.write_yolox_train_config(str(tmp_path / "configs")))
    bt = YT.YoloxTrainBatcher(cfg, str(tmp_path), seed=5, batch_size=8, device=dev)
    try:
        _, targets, _, _ = next(bt)
    finally:
        bt.close()
    assert targets.shape == (8, 120, 5)
    C = 8
    labels = targets.float().cpu()
    assert (labels[..., 0] < C).all() and sum(O.num_labels(labels)) > 8
    xs, ys, es, _, raw = O.make_case(21, 8, 640, C, (0,) * 8)
    outputs = O.decode(raw, xs, ys, es)
    check_case(dev, xs, ys, es, labels, outputs, raw[..., :4], C, True)


@pytest.mark.gpu
def test_conv_weight_gradients(dev):
    """A per-level 1x1 conv with leaf weights, decoded as the head decodes: weight gradients through get_losses match
    those through fp64 autograd of the oracle's loss on the same assignment."""
    from gdrnpp_bop2022_b200 import yolox_loss as Y

    C, B, side, cin = 30, 2, 448, 16
    xs, ys, es, labels, _ = O.make_case(31, B, side, C, (15, 40))
    g = torch.Generator().manual_seed(32)
    feats = [torch.randn(B, cin, side // s, side // s, generator=g) for s in O.STRIDES]
    w0 = torch.randn(5 + C, cin, 1, 1, generator=g) * 0.25
    b0 = torch.randn(5 + C, generator=g) * 0.1
    b0[4:] -= 2.0

    def forward(w, bias, feats, dtype):
        raw = torch.cat([torch.nn.functional.conv2d(f.to(dtype), w, bias).flatten(2).permute(0, 2, 1) for f in feats], 1)
        return O.decode(raw, [t.to(raw) for t in xs], [t.to(raw) for t in ys], [t.to(raw) for t in es]), raw[..., :4]

    grads = []
    # the conv in fp32 (not TF32), with a deterministic weight gradient, so that the reruns can be compared bit for bit
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
        for _ in range(2):
            w = w0.to(dev).requires_grad_(True)
            bias = b0.to(dev).requires_grad_(True)
            out, org = forward(w, bias, [f.to(dev) for f in feats], torch.float32)
            _, L = Y.get_losses(head(C, True), None, [t.to(dev) for t in xs], [t.to(dev) for t in ys],
                                [t.to(dev) for t in es], labels.to(dev), out, levels(org, xs), torch.float32)
            total(L).backward()
            grads.append((w.grad.cpu(), bias.grad.cpu()))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    st = kernel_stages(dev, xs, ys, es, labels, out.detach().cpu(), org.detach().cpu(), C, True)
    w = w0.double().requires_grad_(True)
    bias = b0.double().requires_grad_(True)
    out, org = forward(w, bias, feats, torch.float64)
    cat = lambda ts: torch.cat(ts, 1)[0].double()  # noqa: E731
    li, lo, lc, ll, _ = O.losses_from_assignment(out, org, labels.double(), torch.from_numpy(st["fg"]),
                                                 torch.from_numpy(st["matched"]).long().clamp(min=0),
                                                 torch.from_numpy(st["iou_t"]).double(), cat(xs), cat(ys), cat(es), C, True)
    total(dict(zip(KEYS, (li, lo, lc, ll)))).backward()
    assert rel_err(grads[0][0].double().numpy(), w.grad.numpy()) < 1e-5
    assert rel_err(grads[0][1].double().numpy(), bias.grad.numpy()) < 1e-5
