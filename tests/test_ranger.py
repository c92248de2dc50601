"""Ranger step and model EMA (gdrnpp_bop2022_b200/ranger.py, ema.py, csrc/train_step.cu) against the reference's own
results (tests/golden/ref_ranger.npz, made by tools/make_golden_ref_ranger.py) and the torch-op restatement in
oracle/ranger_oracle.py, in fp32 and fp64."""
import copy
import io
import math
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import ranger_oracle as O

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_ranger.npz")
CHECK_STEPS = (6, 7, 12, 14)
KEYS = ("p",) + O.STATE_KEYS


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _ranger():
    from gdrnpp_bop2022_b200.ranger import Ranger

    return Ranger


def ulp32(x):
    """fp32 ulp at magnitude x."""
    x = max(float(x), 2.0 ** -126)
    return 2.0 ** (math.floor(math.log2(x)) - 23)


def ulp_dist(a, b):
    """Elementwise distance in fp32 ulps (ordered-integer difference)."""
    def ordered(t):
        i = t.contiguous().view(torch.int32).to(torch.int64)
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)

    return (ordered(a) - ordered(b)).abs()


# ------------------------------------------------------------------------------------------------------ CPU
def test_oracle_reproduces_golden_bit_for_bit(golden):
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        for case in O.CASES:
            seen = []

            def on_step(step, groups, opt, case=case, seen=seen):
                if step not in O.GOLDEN_STEPS:
                    return
                vals, steps = O.snapshot(case, groups, opt)
                for (name, key), t in vals.items():
                    t = t.numpy()
                    pre = f"{case}/{step}/{name}/{key}"
                    samp = t.reshape(-1)[O.sample_positions(f"{case}/{name}/{key}", t.shape)]
                    assert np.array_equal(samp, golden[pre + "/samp"]), pre
                    assert t.astype(np.float64).sum() == golden[pre + "/sum"], pre
                assert [steps[n] for n in O.param_names(case)] == golden[f"{case}/{step}/steps"].tolist()
                seen.append(step)

            O.run_case(case, O.RefRanger, torch.float32, "cpu", on_step=on_step)
            assert tuple(seen) == O.GOLDEN_STEPS
    finally:
        torch.set_num_threads(threads)


def test_golden_step_counters_lag_without_gradient(golden):
    steps = golden[f"gdrn/{O.LAST_STEP}/steps"]
    names = O.param_names("gdrn")
    assert steps[names.index("gamma")] == O.LAST_STEP - 2
    assert all(s == O.LAST_STEP for n, s in zip(names, steps) if n != "gamma")


def test_oracle_ema_reproduces_golden(golden):
    for i, (decay, updates) in enumerate(O.EMA_CASES):
        model = O.make_ema_model(seed=i)
        ema_sd = copy.deepcopy(model).state_dict()
        for u in range(3):
            O.perturb_model(model, i, u + 1)
            updates += 1
            O.ema_update(ema_sd, model.state_dict(), O.ema_decay(decay, updates))
        assert updates == int(golden[f"ema{i}/updates"])
        for k, v in ema_sd.items():
            assert np.array_equal(v.numpy(), golden[f"ema{i}/{k}"]), (i, k)


def test_bad_hyper_parameters_raise_reference_errors():
    Ranger = _ranger()
    p = [torch.nn.Parameter(torch.zeros(3))]
    for kw, msg in ((dict(alpha=1.5), "Invalid slow update rate: 1.5"), (dict(k=0), "Invalid lookahead steps: 0"),
                    (dict(lr=0), "Invalid Learning Rate: 0"), (dict(eps=-1.0), "Invalid eps: -1.0")):
        with pytest.raises(ValueError) as e:
            Ranger(p, **kw)
        assert str(e.value) == msg
        with pytest.raises(ValueError) as e2:
            O.RefRanger(p, **kw)
        assert str(e2.value) == msg


def test_constructor_surface_matches_reference():
    Ranger = _ranger()
    p = [torch.nn.Parameter(torch.zeros(3))]
    a, b = Ranger(p, gc_conv_only=True), O.RefRanger(p, gc_conv_only=True)
    assert a.defaults == b.defaults and "step_counter" in a.defaults
    for attr in ("N_sma_threshhold", "alpha", "k", "radam_buffer", "use_gc", "gc_gradient_threshold"):
        assert getattr(a, attr) == getattr(b, attr), attr
    assert not getattr(a, "_step_supports_amp_scaling", False)


def _one(p, g):
    p = torch.nn.Parameter(p)
    p.grad = g
    return p


@pytest.mark.parametrize("make,err,words", [
    (lambda: _one(torch.zeros(4, 3, dtype=torch.float64), torch.zeros(4, 3, dtype=torch.float64)), TypeError,
     "float32"),
    (lambda: _one(torch.zeros(4, 3), torch.zeros(3, 4).t()), ValueError, "strides"),
    (lambda: _one(torch.zeros(3, 4).t(), torch.zeros(3, 4).t()), ValueError, "dim 0 outermost"),
    (lambda: _one(torch.zeros(4, 6)[:, ::2], torch.zeros(4, 6)[:, ::2]), ValueError, "dim 0 outermost"),
    (lambda: _one(torch.zeros(4, 3), torch.zeros(4, 3)), ValueError, "not a CUDA tensor"),
])
def test_restrictions_raise_before_any_change(make, err, words):
    Ranger = _ranger()
    ok = torch.nn.Parameter(torch.zeros(5))   # no gradient: skipped
    bad = make()
    opt = Ranger([{"params": [ok]}, {"params": [bad]}])
    with pytest.raises(err) as e:
        opt.step()
    assert words in str(e.value)
    assert "parameter 0 of param group 1" in str(e.value) and str(tuple(bad.shape)) in str(e.value)
    assert len(opt.state) == 0 and torch.equal(ok.detach(), torch.zeros(5))


def test_sparse_gradient_raises_reference_error():
    p = torch.nn.Parameter(torch.zeros(4, 3))
    p.grad = torch.zeros(4, 3).to_sparse()
    with pytest.raises(RuntimeError, match="Ranger optimizer does not support sparse gradients"):
        _ranger()([p]).step()


# ------------------------------------------------------------------------------------------------------ GPU
def chain(case, cls, dtype, dev, keep=CHECK_STEPS, steps=O.LAST_STEP):
    """Run the case; {step: (values {(name, key): tensor}, counters {name: step}, grads {name: p.grad})}."""
    out, names = {}, O.param_names(case)

    def on_step(step, groups, opt):
        if step in keep:
            vals, counters = O.snapshot(case, groups, opt)
            flat = [p for ps in groups for p in ps]
            out[step] = ({k: v.detach().clone() for k, v in vals.items()}, counters,
                         {n: p.grad.detach().clone() for n, p in zip(names, flat) if p.grad is not None})

    O.run_case(case, cls, dtype, dev, steps=steps, on_step=on_step)
    return out


def bound_check(fused, o32, o64, what):
    """Max abs error of fused against fp64 <= 2 x that of the fp32 oracle + 2 ulp of the largest magnitude."""
    ref = o64.double()
    e_f = (fused.double() - ref).abs().max().item() if ref.numel() else 0.0
    e_32 = (o32.double() - ref).abs().max().item() if ref.numel() else 0.0
    bound = 2 * e_32 + 2 * ulp32(ref.abs().max().item() if ref.numel() else 0.0)
    assert e_f <= bound, (what, e_f, e_32, bound)
    return e_f / bound


@pytest.fixture(scope="module")
def arms(dev):
    """Per case: the fused chain, the fp32 oracle chain and the fp64 oracle chain on the GPU."""
    Ranger = _ranger()
    return {case: (chain(case, Ranger, torch.float32, dev), chain(case, O.RefRanger, torch.float32, dev),
                   chain(case, O.RefRanger, torch.float64, dev)) for case in O.CASES}


@pytest.mark.gpu
def test_tensors_without_gc_within_one_ulp(dev):
    """Every step starts from the fp32 oracle's state, so differences do not compound."""
    Ranger = _ranger()
    report = {}
    for case, spec in O.CASES.items():
        go, ao = O.make_params(case, torch.float32, dev)
        gf, af = O.make_params(case, torch.float32, dev)
        opt_o, opt_f = O.RefRanger(ao, **spec["opt"]), Ranger(af, **spec["opt"])
        fo, ff = [p for ps in go for p in ps], [p for ps in gf for p in ps]
        names = O.param_names(case)
        differ = total = 0
        for step in range(1, O.LAST_STEP + 1):
            with torch.no_grad():
                for po, pf in zip(fo, ff):
                    pf.copy_(po)
                    st = opt_o.state.get(po)
                    if st:
                        opt_f.state[pf] = {"step": st["step"], **{k: st[k].clone() for k in O.STATE_KEYS}}
                    else:
                        opt_f.state.pop(pf, None)
            opt_f.radam_buffer = copy.deepcopy(opt_o.radam_buffer)
            for opt, groups in ((opt_o, go), (opt_f, gf)):
                O.set_lrs(case, opt, step)
                O.set_grads(case, groups, step)
            opt_o.step()
            opt_f.step()
            torch.cuda.synchronize()
            for n, po, pf in zip(names, fo, ff):
                if po.dim() > opt_o.gc_gradient_threshold or not opt_o.state.get(po):
                    continue
                so, sf = opt_o.state[po], opt_f.state[pf]
                assert so["step"] == sf["step"], (case, n, step)
                for a, b, k in [(po.detach(), pf.detach(), "p")] + [(so[k], sf[k], k) for k in O.STATE_KEYS]:
                    d = ulp_dist(a, b)
                    assert d.max().item() <= 1, (case, n, k, step, d.max().item())
                    differ += int((d > 0).sum())
                    total += d.numel()
        report[case] = (differ, total)
    print("elements differing from the fp32 oracle (differ, compared):", report)


@pytest.mark.gpu
def test_accuracy_against_fp64(arms):
    worst = 0.0
    for case, (fu, o32, o64) in arms.items():
        for step in CHECK_STEPS:
            vf, cf, _ = fu[step]
            v32, c32, _ = o32[step]
            v64, c64, _ = o64[step]
            assert cf == c32 == c64, (case, step)
            for key in vf:
                worst = max(worst, bound_check(vf[key], v32[key], v64[key], (case, step, key)))
    print("largest error / bound:", worst)


@pytest.mark.gpu
def test_matches_golden_at_sample_positions(arms, golden):
    for case, (fu, o32, o64) in arms.items():
        for step in set(CHECK_STEPS) & set(O.GOLDEN_STEPS):
            vf, cf, _ = fu[step]
            v32, _, _ = o32[step]
            v64, _, _ = o64[step]
            assert [cf[n] for n in O.param_names(case)] == golden[f"{case}/{step}/steps"].tolist()
            for (name, key), t in vf.items():
                pos = torch.from_numpy(O.sample_positions(f"{case}/{name}/{key}", t.shape)).to(t.device)
                g = torch.from_numpy(golden[f"{case}/{step}/{name}/{key}/samp"]).to(t.device).double()
                ref = v64[(name, key)].reshape(-1).double()
                e_32 = (v32[(name, key)].reshape(-1).double() - ref).abs().max().item()
                bound = 2 * e_32 + 2 * ulp32(ref.abs().max().item())
                e = (t.reshape(-1)[pos].double() - g).abs().max().item()
                assert e <= bound, (case, step, name, key, e, bound)


@pytest.mark.gpu
def test_gradient_is_centralised_in_place(arms):
    for case, (fu, o32, o64) in arms.items():
        for step in CHECK_STEPS:
            gf, g32, g64 = fu[step][2], o32[step][2], o64[step][2]
            assert gf.keys() == g64.keys()
            for n in gf:
                bound_check(gf[n], g32[n], g64[n], (case, step, "grad", n))
    # and GC really happened: the dim-0 slices of a centralised gradient have (about) zero mean
    g = arms["gdrn"][0][14][2]["fc1.weight"]
    assert g.double().mean(dim=1).abs().max().item() < 1e-9


def _state_dict_from_golden(golden, opt):
    sd = opt.state_dict()
    n = len(sd["param_groups"][0]["params"]) + len(sd["param_groups"][1]["params"])
    sd["state"] = {i: {"step": int(golden[f"resume/step/{i}"]),
                       **{k: torch.from_numpy(golden[f"resume/{k}/{i}"].copy()) for k in O.STATE_KEYS}}
                   for i in range(n)}
    return sd


@pytest.mark.gpu
def test_resume_from_reference_state_dict(arms, golden, dev):
    Ranger = _ranger()
    case = O.RESUME_CASE
    groups, arg = O.make_params(case, torch.float32, dev)
    flat = [p for ps in groups for p in ps]
    with torch.no_grad():
        for i, p in enumerate(flat):
            p.copy_(torch.from_numpy(golden[f"resume/p/{i}"]))
    opt = Ranger(arg, **O.CASES[case]["opt"])
    opt.load_state_dict(_state_dict_from_golden(golden, opt))
    for step in range(O.RESUME_STEP + 1, O.LAST_STEP + 1):
        O.set_lrs(case, opt, step)
        O.set_grads(case, groups, step)
        opt.step()
    vals, counters = O.snapshot(case, groups, opt)
    _, o32, o64 = arms[case]
    assert counters == o64[O.LAST_STEP][1]
    for key in vals:
        bound_check(vals[key], o32[O.LAST_STEP][0][key], o64[O.LAST_STEP][0][key], ("resume", key))


@pytest.mark.gpu
def test_state_dict_continues_in_reference_class(arms, dev):
    Ranger = _ranger()
    case = "gdrn"
    spec = O.CASES[case]
    groups, opt = O.run_case(case, Ranger, torch.float32, dev, steps=O.RESUME_STEP)
    sd = copy.deepcopy(opt.state_dict())
    keys = {k for st in sd["state"].values() for k in st}
    assert keys == {"step", *O.STATE_KEYS}
    assert all(type(st["step"]) is int for st in sd["state"].values())
    g2, arg2 = O.make_params(case, torch.float32, dev)
    with torch.no_grad():
        for a, b in zip([p for ps in g2 for p in ps], [p for ps in groups for p in ps]):
            a.copy_(b)
    ref = O.RefRanger(arg2, **spec["opt"])
    ref.load_state_dict(sd)
    for step in range(O.RESUME_STEP + 1, O.LAST_STEP + 1):
        for o, g in ((opt, groups), (ref, g2)):
            O.set_lrs(case, o, step)
            O.set_grads(case, g, step)
            o.step()
    va, ca = O.snapshot(case, groups, opt)
    vb, cb = O.snapshot(case, g2, ref)
    _, o32, o64 = arms[case]
    assert ca == cb == o64[O.LAST_STEP][1]
    for key in va:
        bound_check(vb[key], o32[O.LAST_STEP][0][key], o64[O.LAST_STEP][0][key], ("reference class", key))
        bound_check(va[key], o32[O.LAST_STEP][0][key], o64[O.LAST_STEP][0][key], ("continued", key))
    # torch.save writes each state tensor once, as the reference layout does
    sizes = []
    for o in (opt, ref):
        buf = io.BytesIO()
        torch.save(o.state_dict(), buf)
        sizes.append(buf.tell())
    assert abs(sizes[0] - sizes[1]) <= 0.01 * sizes[1], sizes


def _layout_case(dev, shapes, channels_last=(), steps=7, seed=0):
    """Fused vs fp32 / fp64 oracle on arbitrary shapes; returns the worst error / bound."""
    Ranger = _ranger()
    gen = torch.Generator(device=dev).manual_seed(seed)
    init = [0.05 * torch.randn(s, generator=gen, device=dev) for s in shapes]
    grads = [[1e-2 * torch.randn(s, generator=gen, device=dev) for s in shapes] for _ in range(steps)]

    def arm(cls, dtype):
        ps = []
        for i, x in enumerate(init):
            x = x.to(dtype, copy=True)   # a Parameter shares the storage it is given
            if i in channels_last:
                x = x.contiguous(memory_format=torch.channels_last)
            ps.append(torch.nn.Parameter(x))
        opt = cls(ps, lr=8e-4, weight_decay=0.01)
        for s in range(steps):
            for i, (p, g) in enumerate(zip(ps, grads[s])):
                g = g.to(dtype, copy=True)
                p.grad = g.contiguous(memory_format=torch.channels_last) if i in channels_last else g
            opt.step()
        return ps, opt

    pf, of = arm(Ranger, torch.float32)
    p32, o32 = arm(O.RefRanger, torch.float32)
    p64, o64 = arm(O.RefRanger, torch.float64)
    worst = 0.0
    for i, (a, b, c) in enumerate(zip(pf, p32, p64)):
        if i in channels_last:
            assert a.stride() == b.stride() and of.state[a]["exp_avg"].stride() == a.stride()
        worst = max(worst, bound_check(a.detach(), b.detach(), c.detach(), (i, "p")))
        worst = max(worst, bound_check(a.grad, b.grad, c.grad, (i, "grad")))
        for k in O.STATE_KEYS:
            worst = max(worst, bound_check(of.state[a][k], o32.state[b][k], o64.state[c][k], (i, k)))
    return worst


@pytest.mark.gpu
def test_channels_last_conv_weights(dev):
    _layout_case(dev, [(64, 32, 3, 3), (32, 1, 7, 7), (16, 8, 1, 1)], channels_last=(0, 1, 2))


@pytest.mark.gpu
def test_long_rows_and_many_chunks(dev):
    # [4, 300000]: rows above the on-chip bound; [2048, 2048]: many chunks per tensor; [3, 8193] just above the bound
    _layout_case(dev, [(4, 300000), (2048, 2048), (3, 8193), (5, 8192), (7, 1025), (9, 1024)])


@pytest.mark.gpu
def test_two_thousand_one_element_parameters(dev):
    _layout_case(dev, [(1,)] * 2000 + [(3, 2)], steps=6)


@pytest.mark.gpu
def test_empty_parameters_take_bookkeeping_only(dev):
    Ranger = _ranger()
    e, f = torch.nn.Parameter(torch.zeros(0, 5, device=dev)), torch.nn.Parameter(torch.ones(3, 4, device=dev))
    e.grad, f.grad = torch.zeros(0, 5, device=dev), torch.ones(3, 4, device=dev)
    opt = Ranger([e, f])
    opt.step()
    assert opt.state[e]["step"] == 1 and opt.state[e]["exp_avg"].shape == (0, 5)


@pytest.mark.gpu
def test_launch_count_does_not_depend_on_tensor_count(dev, lib):
    Ranger = _ranger()
    counts = []
    for n in (10, 380):
        ps = [torch.nn.Parameter(torch.randn(8, 16, device=dev)) for _ in range(n)]
        opt = Ranger(ps)
        for step in range(2):
            for p in ps:
                p.grad = torch.randn_like(p)
            before = lib.gdrn_launch_count()
            opt.step()
            counts.append(lib.gdrn_launch_count() - before)
    assert counts == [1, 1, 1, 1], counts


@pytest.mark.gpu
def test_reruns_are_bit_identical(dev):
    Ranger = _ranger()
    a = chain("gdrn", Ranger, torch.float32, dev)
    b = chain("gdrn", Ranger, torch.float32, dev)
    for step in CHECK_STEPS:
        for key in a[step][0]:
            assert torch.equal(a[step][0][key], b[step][0][key]), (step, key)
        for n in a[step][2]:
            assert torch.equal(a[step][2][n], b[step][2][n]), (step, n)


@pytest.mark.gpu
def test_grad_scaler(dev):
    Ranger = _ranger()
    case = "gdrn"
    scaler = torch.amp.GradScaler("cuda")
    g1, a1 = O.make_params(case, torch.float32, dev)
    g2, a2 = O.make_params(case, torch.float32, dev)
    o1, o2 = Ranger(a1, **O.CASES[case]["opt"]), Ranger(a2, **O.CASES[case]["opt"])
    f1, f2 = [p for ps in g1 for p in ps], [p for ps in g2 for p in ps]
    for step in range(1, 8):
        scale = scaler.scale(torch.ones((), device=dev)).item()
        assert scale == 2.0 ** round(math.log2(scale))
        for o, g in ((o1, g1), (o2, g2)):
            O.set_lrs(case, o, step)
            O.set_grads(case, g, step)
        for p in f1:
            if p.grad is not None:
                p.grad.mul_(scale)
        if step == 4:   # an inf gradient: the step is skipped, nothing changes
            before = ([p.detach().clone() for p in f1], copy.deepcopy(o1.state_dict()))
            f1[0].grad[0, 0, 0, 0] = float("inf")
            scaler.step(o1)
            scaler.update()
            assert all(torch.equal(a, p.detach()) for a, p in zip(before[0], f1))
            sd = o1.state_dict()
            for i, st in before[1]["state"].items():
                assert st["step"] == sd["state"][i]["step"]
                for k in O.STATE_KEYS:
                    assert torch.equal(st[k], sd["state"][i][k])
            continue
        scaler.step(o1)
        scaler.update()
        o2.step()
        for a, b in zip(f1, f2):
            assert torch.equal(a.detach(), b.detach()), step
            if a in o1.state and o1.state[a]:
                for k in O.STATE_KEYS:
                    assert torch.equal(o1.state[a][k], o2.state[b][k]), (step, k)
                assert o1.state[a]["step"] == o2.state[b]["step"]


def _full_set(which):
    if which == "gdrn":
        from gdrnpp_bop2022_b200.synthetic import state_dict_shapes

        return list(state_dict_shapes().values()), dict(lr=8e-4, weight_decay=0.01)
    from gdrnpp_bop2022_b200.yolox_model import YOLOX

    return [tuple(p.shape) for p in YOLOX(1.33, 1.25, 8).parameters()], dict(lr=0.001, weight_decay=0)


@pytest.mark.gpu
@pytest.mark.parametrize("which,count", [("gdrn", 380), ("yolox", 456)])
def test_full_parameter_sets_lookahead_step(dev, which, count):
    Ranger = _ranger()
    shapes, kw = _full_set(which)
    assert len(shapes) == count
    gen = torch.Generator(device=dev).manual_seed(7)
    init = [0.02 * torch.randn(s, generator=gen, device=dev) for s in shapes]
    grads = [[1e-3 * torch.randn(s, generator=gen, device=dev) for s in shapes] for _ in range(2)]

    def arm(cls, dtype):
        ps = [torch.nn.Parameter(x.to(dtype, copy=True)) for x in init]
        opt = cls(ps, **kw)
        for step in range(1, 7):   # step 6 is the first lookahead step (k = 6)
            for p, g in zip(ps, grads[step % 2]):
                p.grad = g.to(dtype, copy=True)
            opt.step()
        return ps, opt

    results = {}
    for name, cls, dtype in (("fused", Ranger, torch.float32), ("o32", O.RefRanger, torch.float32),
                             ("o64", O.RefRanger, torch.float64)):
        ps, opt = arm(cls, dtype)
        results[name] = [[p.detach()] + [opt.state[p][k] for k in O.STATE_KEYS] for p in ps]
        del ps, opt
    for i in range(len(shapes)):
        for j, key in enumerate(KEYS):
            bound_check(results["fused"][i][j], results["o32"][i][j], results["o64"][i][j], (which, i, key))


@pytest.mark.gpu
def test_ema_full_yolox_state_bit_exact(dev):
    from gdrnpp_bop2022_b200.ema import ModelEMA
    from gdrnpp_bop2022_b200.yolox_model import YOLOX

    torch.manual_seed(0)
    model = YOLOX(1.33, 1.25, 8).to(dev)
    ema = ModelEMA(model, 0.9998)
    ref = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    assert sum(1 for v in ref.values() if v.is_floating_point()) == 748
    for u in range(1, 4):
        O.perturb_model(model, 5, u)
        ema.update(model)
        O.ema_update(ref, model.state_dict(), O.ema_decay(0.9998, u))
        sd = ema.ema.state_dict()
        for k, v in ref.items():
            assert torch.equal(sd[k], v), (u, k)
    assert ema.updates == 3
    assert not any(p.requires_grad for p in ema.ema.parameters()) and not ema.ema.training


@pytest.mark.gpu
def test_ema_matches_golden(golden, dev):
    from gdrnpp_bop2022_b200.ema import ModelEMA

    for i, (decay, updates) in enumerate(O.EMA_CASES):
        model = O.make_ema_model(seed=i).to(dev)
        ema = ModelEMA(model, decay, updates)
        for u in range(3):
            O.perturb_model(model, i, u + 1)
            ema.update(model)
        assert ema.updates == int(golden[f"ema{i}/updates"])
        for k, v in ema.ema.state_dict().items():
            assert np.array_equal(v.cpu().numpy(), golden[f"ema{i}/{k}"]), (i, k)


@pytest.mark.gpu
def test_ema_rejections(dev):
    from gdrnpp_bop2022_b200.ema import ModelEMA

    model = O.make_ema_model(seed=0).to(dev)
    ema = ModelEMA(model, 0.9998)
    other = torch.nn.Sequential(torch.nn.Conv2d(3, 16, 3, bias=False))
    with pytest.raises(KeyError):
        ema.update(other.to(dev))
    half = copy.deepcopy(model).half()
    with pytest.raises(TypeError, match="0.weight"):
        ema.update(half)
    assert ema.updates == 0
    ema.update_attr(model)
