"""The GDRN training loss (gdrnpp_bop2022_b200/gdrn_loss.py, csrc/gdrn_loss.cu) against the reference's own gdrn_loss
(tests/golden/ref_gdrn_loss.npz, made by tools/make_golden_ref_gdrn_loss.py) and the torch restatement in
oracle/gdrn_loss_oracle.py.

CPU: the fp64 oracle reproduces the golden losses, symmetry choices and gradients; every unsupported option is rejected
by name; the model's forward(do_loss=True) still refuses.  GPU: every kernel stage on its own input (dense partials and
log-sum-exp, the closest symmetric rotation and the point sums, the map gradients by the kernel's fp32 formulas), then
losses and gradients against fp64 autograd and the golden file, bit-identical reruns, label rejection, and a real
GdrnTrainBatcher batch through a small torch head whose parameter gradients match the oracle's.
"""
import os
import pickle

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import gdrn_loss_oracle as O

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_gdrn_loss.npz")
GAP_DEG = 1e-4
KEYS = tuple(O.LOSS_WEIGHTS)
ARGS = ("out_mask_vis", "out_mask_full", "gt_mask_trunc", "gt_mask_visib", "gt_mask_obj", "gt_mask_full", "out_x",
        "out_y", "out_z", "gt_xyz", "gt_xyz_bin", "out_region", "gt_region", "out_rot", "gt_rot", "out_trans",
        "gt_trans", "out_centroid", "out_trans_z", "gt_trans_ratio", "gt_points", "sym_infos", "extents")


def golden(name):
    z = np.load(GOLDEN)
    return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}


def case(name, dtype, device="cpu"):
    ck, cf = O.GOLDEN_CASES[name]
    return O.to(O.make_case(**ck), dtype, device), O.make_cfg(**cf)


def check_against_golden(name, losses, grads, rtol_loss, rtol_grad):
    ref = golden(name)
    want = ref["losses"]
    got = np.array([float(losses[k].detach()) if k in losses else np.nan for k in KEYS])
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_allclose(got[ok], want[ok], rtol=rtol_loss, atol=1e-7)
    for k in O.SMALL:
        g = grads.get(k)
        g = np.zeros_like(ref["grad_" + k]) if g is None else g
        np.testing.assert_allclose(g, ref["grad_" + k], rtol=0, atol=rtol_grad * max(np.abs(ref["grad_" + k]).max(), 1e-30))
    for k in O.DENSE:
        g = grads.get(k)
        g = np.zeros(1) if g is None else g
        s = ref["gsamp_" + k]
        got_s = g.reshape(-1)[O.sample_positions(k, g.shape)] if g.size > 1 else np.zeros_like(s)
        np.testing.assert_allclose(got_s, s, rtol=0, atol=rtol_grad * max(np.abs(s).max(), 1e-30))


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(O.GOLDEN_CASES))
def test_oracle_reproduces_reference(name):
    d, cfg = case(name, torch.float64)
    rec = {}
    losses = O.gdrn_loss(cfg, d, model=O.MtlModel(), record=rec)
    O.weighted_total(losses).backward()
    grads = {k: d[k].grad.numpy() for k in O.DENSE + O.SMALL if d[k].grad is not None}
    # the reference runs in fp32: its region sum over 10^5 pixels and its PM sum carry ~1e-6 of rounding
    check_against_golden(name, losses, grads, 2e-5, 1e-4)
    ref = golden(name)
    if "sym_idx" in rec:
        sure = ref["sym_gap"] > GAP_DEG
        np.testing.assert_array_equal(rec["sym_idx"][sure], ref["sym_idx"][sure])


def test_golden_cases_have_decisive_choices():
    """Most symmetric ROIs of the golden cases are decided by a clear margin, so the index comparison has teeth."""
    gaps = np.concatenate([golden(n)["sym_gap"] for n in O.GOLDEN_CASES])
    fin = gaps[np.isfinite(gaps)]
    assert len(fin) > 40 and (fin > GAP_DEG).mean() > 0.9


@pytest.mark.parametrize("option, value", [
    ("XYZ_LOSS_TYPE", "CE_coor"), ("MASK_LOSS_TYPE", "RW_BCE"), ("MASK_LOSS_TYPE", "dice"), ("MASK_LOSS_TYPE", "CE"),
    ("FULL_MASK_LOSS_TYPE", "CE"), ("REGION_LOSS_TYPE", "BCE"), ("PM_R_ONLY", False), ("PM_LOSS_TYPE", "Smooth_L1"),
    ("CENTROID_LOSS_TYPE", "MSE"), ("Z_LOSS_TYPE", "L2"), ("ROT_LW", 1.0), ("TRANS_LW", 1.0), ("BIND_LW", 1.0),
    ("XYZ_LOSS_MASK_GT", "full"), ("Z_TYPE", "LOG")])
def test_rejects_unsupported_options(option, value):
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    cfg = O.make_cfg(z_type=value) if option == "Z_TYPE" else O.make_cfg(**{option: value})
    with pytest.raises(NotImplementedError, match=option):
        G.check_cfg(cfg)


def test_rejects_quaternion_gt_rot_and_cpu_tensors():
    from gdrnpp_bop2022_b200 import _lib
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    d = O.to(O.make_case(0, 2), torch.float32, grad=False)
    args = {k: d[k] for k in ARGS}
    cfg = O.make_cfg(freeze=True, CENTROID_LW=0.0, Z_LW=0.0)
    with pytest.raises(NotImplementedError, match="quaternion"):
        G.gdrn_loss(None, cfg, **{**args, "gt_rot": torch.zeros(2, 4)})
    with pytest.raises(_lib.GdrnError, match="CUDA"):
        G.gdrn_loss(None, O.make_cfg(), **args)


def test_check_cfg_keys_follow_the_reference():
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    assert G.check_cfg(O.make_cfg()).keys == list(KEYS)
    assert G.check_cfg(O.make_cfg(freeze=True)).keys == ["loss_PM_R", "loss_centroid", "loss_z"]
    assert "loss_mask_full" not in G.check_cfg(O.make_cfg(FULL_MASK_LW=0.0)).keys
    assert G.check_cfg(O.make_cfg(XYZ_LW=0.0)).keys[0] == "loss_coor_x"   # present at weight 0, as the reference


def test_forward_do_loss_still_refuses():
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg

    m = GDRN_DoubleMask(default_cfg(), max_batch=1)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 256, 256), do_loss=True)


# ------------------------------------------------------------------------------------------------------------ GPU
def ulp_close(got, want, n=1):
    got, want = got.float().cpu().numpy(), want.float().cpu().numpy()
    tol = n * np.spacing(np.maximum(np.abs(want), np.abs(got)).astype(np.float32))
    bad = np.abs(got.astype(np.float64) - want.astype(np.float64)) > tol
    assert not bad.any(), (bad.sum(), got[bad][:5], want[bad][:5])


def run_gpu(cfg, d, model=None):
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    losses = G.gdrn_loss(model, cfg, **{k: d[k] for k in ARGS})
    O.weighted_total(losses).backward()
    grads = {k: d[k].grad.detach().clone() for k in O.DENSE + O.SMALL if d[k].grad is not None}
    return losses, grads


def stages(cfg, d):
    """Forward stages of one call, read back from the workspace."""
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    plan = G.check_cfg(cfg)
    losses = G.gdrn_loss(O.MtlModel(torch.float32, d["out_x"].device), cfg, **{k: d[k] for k in ARGS})
    fn = next(iter(losses.values())).grad_fn
    while fn is not None and not hasattr(fn, "ws"):
        fn = fn.next_functions[0][0]
    B, HW = d["out_rot"].shape[0], d["out_x"].shape[2] * d["out_x"].shape[3]
    _, offs = G.workspace_layout(B, HW)
    v = lambda n, dt, sh: G.workspace_view(fn.ws, offs, n, dt, sh)  # noqa: E731
    tiles = (HW + O.TILE - 1) // O.TILE
    return plan, fn, {"partial": v("partial", torch.float64, (B * tiles, 8)), "lse": v("lse", torch.float32, (B, HW)),
                      "sym_idx": v("sym_idx", torch.int32, (B,)), "rot_sel": v("rot_sel", torch.float32, (B, 3, 3)),
                      "pm_abs": v("pm_abs", torch.float64, (B,)), "pm_sign": v("pm_sign", torch.float64, (B, 3, 3)),
                      "norm": v("norm", torch.float32, (4,)), "tiles": tiles}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["b1", "b8_two_bce", "b48_mixed", "b36_cont_mtl", "b3_empty"])
def test_stages(dev, name):
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    d, cfg = case(name, torch.float32, dev)
    plan, fn, st = stages(cfg, d)
    d = {k: v.detach() if torch.is_tensor(v) else v for k, v in d.items()}
    # stage 1: per-CTA partials and the per-pixel log-sum-exp
    want = O.replay_partials(cfg, d, st["tiles"]).cpu()
    got = st["partial"].cpu()
    if not plan.flags & G.F_FULL:
        want[:, 4] = 0
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-6, atol=1e-4)
    np.testing.assert_allclose(st["lse"].cpu().numpy(), O.replay_lse(cfg, d).cpu().numpy(), rtol=2e-7, atol=4e-6)
    # stage 2: the closest symmetric rotation (fp64 choice wherever its gap is decisive) and the point sums
    syms = d["sym_infos"] if cfg.MODEL.POSE_NET.LOSS_CFG.PM_LOSS_SYM else [None] * len(d["sym_infos"])
    idx, rots, gap = O.replay_closest(d["out_rot"], d["gt_rot"], syms)
    sure = gap > GAP_DEG
    np.testing.assert_array_equal(st["sym_idx"].cpu().numpy()[sure], idx[sure])
    np.testing.assert_allclose(st["rot_sel"].cpu().numpy()[sure], rots.numpy()[sure], rtol=0, atol=1e-6)
    ext = d["extents"].max(1)[0]
    w = 1.0 / ext if cfg.MODEL.POSE_NET.LOSS_CFG.PM_NORM_BY_EXTENT else torch.ones_like(ext)
    pm_abs, pm_sign, n_near = O.replay_pm_sums(d["out_rot"], st["rot_sel"], d["gt_points"], w)
    np.testing.assert_allclose(st["pm_abs"].cpu().numpy(), pm_abs.cpu().numpy(), rtol=1e-6)
    wp = (w.view(-1, 1, 1) * d["gt_points"].abs()).amax((1, 2)).double()
    bound = (2 * n_near.double() * wp + 1e-7 * wp * d["gt_points"].shape[1]).view(-1, 1, 1)
    assert ((st["pm_sign"] - pm_sign).abs() <= bound).all()
    # stage 4: the map gradients by the kernel's formulas from its own log-sum-exp and normalisers
    up = torch.tensor([O.LOSS_WEIGHTS[k] for k in KEYS], dtype=torch.float32, device=dev)
    grads = G.backward_raw(fn.inp, fn.ws, up)
    want = O.replay_map_grads(cfg, d, st["lse"], st["norm"], up)
    for i, k in enumerate(("out_x", "out_y", "out_z", "out_mask_vis", "out_mask_full", "out_region")):
        if k in want:
            ulp_close(grads[i], want[k])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(O.GOLDEN_CASES))
def test_losses_and_gradients(dev, name):
    d32, cfg = case(name, torch.float32, dev)
    model = O.MtlModel(torch.float32, dev)
    losses, grads = run_gpu(cfg, d32, model)
    # fp64 oracle on the same fp32 inputs
    d64, _ = case(name, torch.float64)
    m64 = O.MtlModel()
    want = O.gdrn_loss(cfg, d64, model=m64)
    O.weighted_total(want).backward()
    assert set(losses) == set(want)
    for k in want:
        assert losses[k].dtype == torch.float32 and losses[k].dim() == 0 and losses[k].is_cuda
        np.testing.assert_allclose(float(losses[k].detach()), float(want[k].detach()), rtol=1e-6, atol=1e-9)
    if cfg.MODEL.POSE_NET.USE_MTL:
        for k in want:
            lv = k.replace("loss_", "log_var_")
            np.testing.assert_allclose(float(getattr(model, lv).grad), float(getattr(m64, lv).grad), rtol=1e-5)
    # dense gradients against fp64 autograd: fp32 rounding of the scale and the softmax
    for k in O.DENSE:
        if d64[k].grad is None:
            assert k not in grads
            continue
        g, r = grads[k].double().cpu(), d64[k].grad
        assert (g - r).abs().max() <= 1e-5 * r.abs().max() + 1e-12, k
    # small gradients: out_rot up to the sign flips of points whose fp32 difference is within 1e-6 of 0
    for k in ("out_centroid", "out_trans_z"):
        if d64[k].grad is not None:
            np.testing.assert_allclose(grads[k].cpu().numpy(), d64[k].grad.numpy(), rtol=1e-6, atol=1e-12)
    if d64["out_rot"].grad is not None:
        lc = cfg.MODEL.POSE_NET.LOSS_CFG
        syms = d64["sym_infos"] if lc.PM_LOSS_SYM else [None] * len(d64["sym_infos"])
        _, rots, _ = O.replay_closest(d64["out_rot"], d64["gt_rot"], syms)
        ext = d64["extents"].max(1)[0]
        w = 1.0 / ext if lc.PM_NORM_BY_EXTENT else torch.ones_like(ext)
        _, _, n_near = O.replay_pm_sums(d64["out_rot"].detach(), rots, d64["gt_points"], w)
        B, N = d64["gt_points"].shape[:2]
        scale = 3 * lc.PM_LW * O.LOSS_WEIGHTS["loss_PM_R"] / (B * N * 3)
        if cfg.MODEL.POSE_NET.USE_MTL:
            scale *= float(torch.exp(-m64.log_var_PM_R.detach()))
        wp = (w.view(-1, 1, 1) * d64["gt_points"].abs()).amax((1, 2))
        bound = scale * (2 * n_near * wp + 1e-5 * N * wp).view(-1, 1, 1)
        assert ((grads["out_rot"].double().cpu() - d64["out_rot"].grad).abs() <= bound).all()
    # end to end against the reference's own fp32 run
    check_against_golden(name, losses, {k: v.cpu().numpy() for k, v in grads.items()}, 2e-5, 1e-4)
    # two runs are bit-identical
    d2, _ = case(name, torch.float32, dev)
    losses2, grads2 = run_gpu(cfg, d2, O.MtlModel(torch.float32, dev))
    for k in losses:
        assert torch.equal(losses[k], losses2[k])
    for k in grads:
        assert torch.equal(grads[k], grads2[k])


@pytest.mark.gpu
def test_strided_head_outputs(dev):
    """Channel slices of one [B,3,H,W] coordinate output (the head's layout) give the contiguous result."""
    d, cfg = case("b8_two_bce", torch.float32, dev)
    want, gwant = run_gpu(cfg, d)
    coor = torch.cat([d["out_x"], d["out_y"], d["out_z"]], 1).detach().requires_grad_(True)
    d2, _ = case("b8_two_bce", torch.float32, dev)
    d2.update(out_x=coor[:, 0:1], out_y=coor[:, 1:2], out_z=coor[:, 2:3])
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    got = G.gdrn_loss(None, cfg, **{k: d2[k] for k in ARGS})
    O.weighted_total(got).backward()
    for k in want:
        assert torch.equal(got[k], want[k])
    assert torch.equal(coor.grad, torch.cat([gwant["out_x"], gwant["out_y"], gwant["out_z"]], 1))


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [65, -1])
def test_region_label_out_of_range_is_rejected(dev, bad):
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    d, cfg = case("b1", torch.float32, dev)
    m = d["gt_mask_visib"][0].nonzero()[0]
    d["gt_region"][0, m[0], m[1]] = bad
    with pytest.raises(ValueError, match="gt_region"):
        G.gdrn_loss(None, cfg, **{k: d[k] for k in ARGS})
    # outside the region mask the label is multiplied by 0, as in the reference
    d, cfg = case("b1", torch.float32, dev)
    m = (d["gt_mask_visib"][0] == 0).nonzero()[0]
    d["gt_region"][0, m[0], m[1]] = bad
    G.gdrn_loss(None, cfg, **{k: d[k] for k in ARGS})


@pytest.mark.gpu
def test_symmetry_tables_upload_once(dev):
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    d, cfg = case("b48_mixed", torch.float32, dev)
    run_gpu(cfg, d)
    table = G._SYM_TABLE[str(d["out_rot"].device)]
    d2 = O.to(O.make_case(seed=9, B=48, syms=("cont", "none", "two"), tables=O.sym_tables()), torch.float32, dev)
    d2["sym_infos"] = d["sym_infos"]
    run_gpu(cfg, d2)
    assert G._SYM_TABLE[str(d["out_rot"].device)] is table


@pytest.mark.gpu
def test_train_batcher_batch_through_a_torch_head(dev, tmp_path):
    """A real GdrnTrainBatcher batch and a small torch head in front of the loss: parameter gradients match the
    oracle's fp64 autograd through the same head."""
    from gdrnpp_bop2022_b200 import train_batch as TB
    from gdrnpp_bop2022_b200.synthetic import write_bop_train_tree
    from gdrnpp_bop2022_b200 import gdrn_loss as G

    from gdrnpp_bop2022_b200.ply import load_ply
    from gdrnpp_bop2022_b200.synthetic import shipped_train_cfg

    root = str(tmp_path)
    base = write_bop_train_tree(root, num_images=4, num_scenes=1, insts_per_image=3, seed=5)
    fps = {}
    for o in (1, 2, 3):   # any points do as region centres here
        pts = load_ply(os.path.join(base, "models", "obj_{:06d}.ply".format(o)), vertex_scale=0.001)["pts"]
        fps[str(o)] = {f"fps{n}_and_center": np.concatenate([pts[np.arange(n) % len(pts)], pts.mean(0, keepdims=True)])
                       for n in TB.FPS_COUNTS}
    with open(os.path.join(base, "models", "fps_points.pkl"), "wb") as f:
        pickle.dump(fps, f)
    batcher = TB.GdrnTrainBatcher(shipped_train_cfg(), root, device=dev, batch_size=6)
    try:
        batch = next(iter(batcher))
    finally:
        batcher.close()
    assert any(s is not None for s in batch["sym_info"])
    B = batch["roi_img"].shape[0]
    R1 = 65

    def head(params, img, ego_rot):
        conv, lin = params
        feat = torch.nn.functional.avg_pool2d(img, img.shape[-1] // 64)
        maps = torch.nn.functional.conv2d(feat, conv)
        pooled = feat.mean((2, 3))
        v = pooled @ lin
        return {"out_x": maps[:, 0:1], "out_y": maps[:, 1:2], "out_z": maps[:, 2:3], "out_mask_vis": maps[:, 3:4],
                "out_mask_full": maps[:, 4:5], "out_region": maps[:, 5:5 + R1],
                "out_rot": ego_rot.to(v.dtype) + 0.1 * v[:, :9].view(B, 3, 3), "out_centroid": v[:, 9:11],
                "out_trans_z": 1.0 + v[:, 11]}

    g = torch.Generator().manual_seed(0)
    conv = torch.randn(5 + R1, 3, 1, 1, generator=g) * 0.5
    lin = torch.randn(3, 12, generator=g) * 0.2
    cfg = O.make_cfg(PM_NORM_BY_EXTENT=True)
    tgt = {"gt_mask_trunc": batch["roi_mask_trunc"], "gt_mask_visib": batch["roi_mask_visib"],
           "gt_mask_obj": batch["roi_mask_obj"], "gt_mask_full": batch["roi_mask_full"], "gt_xyz": batch["roi_xyz"],
           "gt_xyz_bin": None, "gt_region": batch["roi_region"], "gt_rot": batch["ego_rot"], "out_trans": None,
           "gt_trans": batch["trans"], "gt_trans_ratio": batch["roi_trans_ratio"], "gt_points": batch["roi_points"],
           "sym_infos": batch["sym_info"], "extents": batch["roi_extent"]}
    grads = {}
    for dtype, device in ((torch.float32, dev), (torch.float64, "cpu")):
        params = [conv.to(device, dtype).requires_grad_(True), lin.to(device, dtype).requires_grad_(True)]
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):   # the head in true fp32, as the oracle's
            out = head(params, batch["roi_img"].to(device, dtype), batch["ego_rot"].to(device, dtype))
        d = {**{k: v.to(device, dtype) if torch.is_tensor(v) and v.is_floating_point() else v for k, v in tgt.items()},
             **out}
        d["gt_region"] = d["gt_region"].to(device)
        if dtype == torch.float32:
            losses = G.gdrn_loss(None, cfg, **{k: d[k] for k in ARGS})
        else:
            losses = O.gdrn_loss(cfg, d)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            O.weighted_total(losses).backward()
        grads[dtype] = [p.grad.double().cpu() for p in params]
    for got, want in zip(grads[torch.float32], grads[torch.float64]):
        assert (got - want).abs().max() <= 1e-4 * want.abs().max(), ((got - want).abs().max(), want.abs().max())
