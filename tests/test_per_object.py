"""Per-object (class-agnostic) models: the one-slab geometry head through every layer, and PerObjectGDRN, which sends
each ROI of a mixed batch to its object's network."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import gdrn_model_oracle as O
from test_oracle_pinning import _ref_heads_state_dict

GOLD = os.path.join(ROOT, "tests", "golden")
MAPS = ("mask", "full_mask", "coor_x", "coor_y", "coor_z", "region")

BASE_CFG = (   # the defaults of configs/_base_/gdrn_base.py that the hot path reads
    "MODEL = dict(PIXEL_MEAN=[0, 0, 0], PIXEL_STD=[255.0, 255.0, 255.0], POSE_NET=dict(NAME='GDRN', NUM_CLASSES=13,\n"
    "    OUTPUT_RES=64, BACKBONE=dict(INIT_CFG=dict(type='timm/resnet34')),\n"
    "    GEO_HEAD=dict(NUM_REGIONS=64, XYZ_CLASS_AWARE=False, MASK_CLASS_AWARE=False, REGION_CLASS_AWARE=False,\n"
    "                  MASK_THR_TEST=0.5),\n"
    "    PNP_NET=dict(ROT_TYPE='allo_rot6d', TRANS_TYPE='centroid_z', Z_TYPE='REL', REGION_ATTENTION=True,\n"
    "                 WITH_2D_COORD=True)))\n"
    "TEST = dict(USE_PNP=False, SAVE_RESULTS_ONLY=False, USE_DEPTH_REFINE=False, DEPTH_REFINE_ITER=2)\n"
    "INPUT = dict(DZI_PAD_SCALE=1.5)\n")
OBJ_CFG = (    # the shape of configs/gdrn/ycbvSO/convnext_*/002_master_chef_can.py (no class-aware flags of its own)
    "_base_ = ['../_base_/gdrn_base.py']\n"
    "OUTPUT_DIR = 'output/gdrn/ycbvSO/convnext/002_master_chef_can'\n"
    "MODEL = dict(LOAD_DETS_TEST=True, POSE_NET=dict(NAME='GDRN_double_mask', XYZ_ONLINE=True,\n"
    "    BACKBONE=dict(FREEZE=False, INIT_CFG=dict(type='timm/convnext_base', pretrained=True, features_only=True,\n"
    "                                              out_indices=(3,))),\n"
    "    GEO_HEAD=dict(INIT_CFG=dict(type='TopDownDoubleMaskXyzRegionHead', in_dim=1024), NUM_REGIONS=64),\n"
    "    PNP_NET=dict(REGION_ATTENTION=True, WITH_2D_COORD=True, ROT_TYPE='allo_rot6d', TRANS_TYPE='centroid_z')))\n")


def _write_obj_config(tmp_path):
    (tmp_path / "_base_").mkdir(exist_ok=True)
    (tmp_path / "_base_" / "gdrn_base.py").write_text(BASE_CFG)
    (tmp_path / "ycbvSO").mkdir(exist_ok=True)
    p = tmp_path / "ycbvSO" / "002_master_chef_can.py"
    p.write_text(OBJ_CFG)
    return str(p)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_agnostic_head_oracle_matches_reference_classes():
    """ref_heads_agnostic.npz: the reference's TopDownDoubleMaskXyzRegionHead with mask / xyz / region_num_classes = 1
    (tools/make_golden_ref_heads.py --agnostic).  The oracle's one-slab head reads vis 0, full 1, x/y/z 2..4 and
    region 5..69 of the 70-channel out_layer."""
    g = np.load(os.path.join(GOLD, "ref_heads_agnostic.npz"))
    assert int(g["num_classes"]) == 1
    sd = _ref_heads_state_dict(g)
    assert tuple(sd["geo_head_net.out_layer.weight"].shape) == (70, 32, 1, 1)
    with torch.no_grad():
        outs = O.geo_head(sd, torch.from_numpy(g["in/feat"]), num_classes=1)
    for name, o in zip(("vis", "full", "cx", "cy", "cz", "region"), outs):
        ref = torch.from_numpy(g["out/" + name])
        assert o.shape == ref.shape and torch.allclose(o, ref, atol=2e-5, rtol=1e-4), name
    with torch.no_grad():
        rot, t = O.conv_pnp_net(sd, torch.from_numpy(g["in/coor_feat"]), torch.from_numpy(g["in/region"]),
                                torch.from_numpy(g["in/extents"]))
    assert torch.allclose(rot, torch.from_numpy(g["out/pnp_rot"]), atol=1e-5, rtol=1e-4)
    assert torch.allclose(t, torch.from_numpy(g["out/pnp_t_raw"]), atol=1e-5, rtol=1e-4)


def _agnostic_oracle_forward(sd, batch, arch="convnext_base"):
    """GDRN_DoubleMask.forward of a class-agnostic model (GDRN_double_mask.py:96-214 with the three class gathers of
    :107-126 skipped, as they are when XYZ/MASK/REGION_CLASS_AWARE are false), composed of the oracle's pieces.  The
    one-slab head's six views are read directly; roi_classes is not read."""
    import torch.nn.functional as F

    feat = O.convnext_features(sd, batch["roi_img"], arch)
    vis, full, cx, cy, cz, region = O.geo_head(sd, feat, num_classes=1)
    coor_feat = torch.cat([cx, cy, cz, batch["roi_coord_2d"]], dim=1)
    rot6, t_ = O.conv_pnp_net(sd, coor_feat, F.softmax(region[:, 1:], dim=1), batch["roi_extents"])
    rot_m = O.rot6d_to_mat_batch(rot6)
    ego_rot, trans = O.pose_from_predictions_test(rot_m, t_[:, :2], t_[:, 2:3], batch["roi_cams"], batch["roi_centers"],
                                                  batch["resize_ratios"], batch["roi_whs"])
    return {"rot": ego_rot, "trans": trans, "mask": vis, "full_mask": full, "coor_x": cx, "coor_y": cy, "coor_z": cz,
            "region": region, "conv_feat": feat, "rot6d": rot6, "t_": t_}


def test_agnostic_oracle_forward_matches_the_oracle_glue():
    """With one class slab, the oracle's class-aware forward at label 0 gathers the identity: the class-agnostic
    forward above must equal it exactly, for any labels it is given (they are not read)."""
    from gdrnpp_bop2022_b200.synthetic import make_batch, make_state_dict

    sd = make_state_dict(arch="convnext_tiny", num_classes=1, seed=3)
    batch = make_batch(B=2, seed=3)
    with torch.no_grad():
        a = _agnostic_oracle_forward(sd, dict(batch, roi_classes=torch.tensor([7, 400])), arch="convnext_tiny")
        ref = O.gdrn_forward(sd, dict(batch, roi_classes=torch.zeros(2, dtype=torch.int64)), arch="convnext_tiny",
                             num_classes=1, return_maps=True, return_intermediate=True)
    assert a["region"].shape == (2, 65, 64, 64) and a["mask"].shape == (2, 1, 64, 64)
    for k in MAPS + ("rot", "trans", "rot6d", "t_"):
        assert torch.equal(a[k], ref[k]), k


def test_per_object_config_loads_and_builds(tmp_path):
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, build_model_optimizer, load_py_config

    cfg = load_py_config(_write_obj_config(tmp_path))
    pn = cfg.MODEL.POSE_NET
    # inherited from the base: NUM_CLASSES, the three class-aware flags (False), Z_TYPE, TEST / INPUT defaults
    assert pn.NAME == "GDRN_double_mask" and pn.NUM_CLASSES == 13 and pn.PNP_NET.Z_TYPE == "REL"
    assert pn.GEO_HEAD.XYZ_CLASS_AWARE is False and pn.GEO_HEAD.MASK_THR_TEST == 0.5
    assert pn.GEO_HEAD.INIT_CFG.in_dim == 1024 and cfg.TEST.DEPTH_REFINE_ITER == 2 and cfg.INPUT.DZI_PAD_SCALE == 1.5
    assert cfg.MODEL.LOAD_DETS_TEST is True and cfg.MODEL.PIXEL_STD[0] == 255.0
    model, opt = build_model_optimizer(cfg)
    assert opt is None and model.arch == "convnext_base" and model.class_aware is False and model.head_classes == 1
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert shapes["geo_head_net.out_layer.weight"] == (70, 256, 1, 1)
    assert shapes["geo_head_net.out_layer.bias"] == (70,)
    from gdrnpp_bop2022_b200.synthetic import state_dict_shapes

    assert shapes == state_dict_shapes("convnext_base", 1)
    # mixed class-awareness stays out of scope
    (tmp_path / "ycbvSO" / "mixed.py").write_text(
        "_base_ = './002_master_chef_can.py'\nMODEL = dict(POSE_NET=dict(GEO_HEAD=dict(XYZ_CLASS_AWARE=True)))\n")
    mixed = load_py_config(str(tmp_path / "ycbvSO" / "mixed.py"))
    assert mixed.MODEL.POSE_NET.NAME == "GDRN_double_mask" and mixed.MODEL.POSE_NET.GEO_HEAD.MASK_CLASS_AWARE is False
    with pytest.raises(NotImplementedError):
        GDRN_DoubleMask(mixed)
    with pytest.raises(NotImplementedError):
        build_model_optimizer(mixed)


@pytest.mark.parametrize("labels", [
    [4, 1, 4, 9, 1, 1, 9, 4, 2, 9, 2, 4],     # shuffled
    [7],                                      # a single ROI
    [3, 3, 3, 3],                             # one label only
    [5, 0, 2, 8, 1],                          # all distinct
    [],                                       # no detections
])
def test_group_rois_restores_input_order(labels):
    from gdrnpp_bop2022_b200.per_object import group_rois

    known = {0, 1, 2, 3, 4, 5, 7, 8, 9}
    groups = group_rois(torch.tensor(labels, dtype=torch.int64), known)
    lab = np.asarray(labels, np.int64)
    assert [g[0] for g in groups] == sorted(set(labels))
    seen = torch.cat([idx for _, idx in groups]) if groups else torch.zeros(0, dtype=torch.int64)
    assert sorted(seen.tolist()) == list(range(len(labels)))            # every ROI exactly once
    for label, idx in groups:
        assert idx.dtype == torch.int64 and (lab[idx.numpy()] == label).all()
        assert (np.diff(idx.numpy()) > 0).all()                          # input order inside a group
    # scatter of the per-group results (here: a tag per ROI) restores the input order exactly
    payload = torch.arange(len(labels), dtype=torch.float32) * 10 + 3
    out = torch.full((len(labels),), -1.0)
    for _, idx in groups:
        out.index_copy_(0, idx, payload[idx])
    assert torch.equal(out, payload)
    # a plain list gives the same groups as a tensor
    assert [(u, i.tolist()) for u, i in group_rois(list(labels), known)] == [(u, i.tolist()) for u, i in groups]


def test_group_rois_missing_label_raises_and_names_it():
    from gdrnpp_bop2022_b200.per_object import group_rois

    with pytest.raises(ValueError, match=r"\[6, 11\]"):
        group_rois([1, 6, 1, 11, 6], {1, 2})


def test_per_object_members_are_checked():
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg
    from gdrnpp_bop2022_b200.per_object import PerObjectGDRN

    def agnostic(**kw):
        cfg = default_cfg(arch="convnext_tiny")
        g = cfg.MODEL.POSE_NET.GEO_HEAD
        g.XYZ_CLASS_AWARE = g.MASK_CLASS_AWARE = g.REGION_CLASS_AWARE = False
        return GDRN_DoubleMask(cfg, arch="convnext_tiny", **kw)

    a = agnostic(precision="bf16x3")
    with pytest.raises(ValueError, match="class-aware"):
        PerObjectGDRN({0: a, 1: GDRN_DoubleMask(default_cfg(arch="convnext_tiny"), arch="convnext_tiny")})
    with pytest.raises(ValueError, match="precision"):
        PerObjectGDRN({0: a, 1: agnostic(precision="bf16")})
    with pytest.raises(ValueError):
        PerObjectGDRN({})
    pm = PerObjectGDRN({3: a})
    assert pm.precision == "bf16x3" and list(pm.members) == [3]


# ------------------------------------------------------------------------------------------------------------ GPU
def _agnostic_cfg(with_maps=True, arch="convnext_base"):
    from gdrnpp_bop2022_b200.gdrn_model import default_cfg

    cfg = default_cfg(arch=arch, with_maps=with_maps)
    g = cfg.MODEL.POSE_NET.GEO_HEAD
    g.XYZ_CLASS_AWARE = g.MASK_CLASS_AWARE = g.REGION_CLASS_AWARE = False
    return cfg


def _member(dev, seed, precision="bf16x3", max_batch=64, with_maps=True):
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    m = GDRN_DoubleMask(_agnostic_cfg(with_maps), max_batch=max_batch, precision=precision)
    m.load_state_dict(make_state_dict(num_classes=1, seed=seed))
    return m.to(dev)


def _kw(b, roi_classes="keep"):
    return dict(roi_classes=b.get("roi_classes") if roi_classes == "keep" else roi_classes,
                roi_coord_2d=b["roi_coord_2d"], roi_cams=b["roi_cams"], roi_centers=b["roi_centers"],
                roi_whs=b["roi_whs"], roi_extents=b["roi_extents"], resize_ratios=b["resize_ratios"])


def _rot_err(Ra, Rb):
    d = (Ra.double() - Rb.double()).flatten(1).norm(dim=1)
    return 2 * torch.asin((d / (2 * 2 ** 0.5)).clamp(max=1.0))


def _rot6d_conditioning(rot6d):
    """Gram-Schmidt amplification of rot6d -> R, as in test_gpu_parity.py."""
    a1, a2 = rot6d[:, :3].double(), rot6d[:, 3:].double()
    n1 = a1.norm(dim=1)
    x = a1 / n1[:, None]
    a2p = a2 - (a2 * x).sum(1, keepdim=True) * x
    return 1.0 / torch.minimum(n1, a2p.norm(dim=1))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [5, 64])
def test_agnostic_forward_vs_oracle(dev, B):
    """A class-agnostic convnext_base against the class-agnostic fp32 oracle.  bf16x3: the north-star bars of
    test_forward_vs_oracle_north_star_tolerance / _b64 (t < 1e-3, raw rot6d / t_ < 1e-4, maps < 2e-3, R < 1e-4 rad x
    max(1, kappa)); these weights are a different random draw from the bench batch's, so R is scaled by the oracle
    rot6d's conditioning kappa at both sizes (the largest on H100: 2.3 at B = 5, 44 at B = 64, one ROI with a short
    first rot6d column).  bf16: that mode's documented tolerances, R scaled by kappa in the same way."""
    from gdrnpp_bop2022_b200.synthetic import make_batch, make_state_dict

    sd = make_state_dict(num_classes=1, seed=21)
    batch = make_batch(B=B, seed=300 + B)
    with torch.no_grad():
        ref = _agnostic_oracle_forward(sd, batch)
    kappa = _rot6d_conditioning(ref["rot6d"]).clamp_min(1.0)
    print(f"B={B}: largest kappa of the oracle rot6d {kappa.max().item():.3f}")
    gb = {k: v.to(dev) for k, v in batch.items()}
    for precision in ("bf16x3", "bf16"):
        m = _member(dev, 21, precision=precision)
        out = m(gb["roi_img"], return_raw=True, **_kw(gb, roi_classes=None))
        torch.cuda.synchronize()
        raw = out["raw"].cpu()
        rerr = _rot_err(out["rot"].cpu(), ref["rot"])
        terr = (out["trans"].cpu() - ref["trans"]).abs().max().item()
        if precision == "bf16x3":
            for k in MAPS:
                assert (out[k].cpu() - ref[k]).abs().max().item() < 2e-3, k
            assert (raw[:, :6] - ref["rot6d"]).abs().max().item() < 1e-4
            assert (raw[:, 6:] - ref["t_"]).abs().max().item() < 1e-4
            assert (rerr < 1e-4 * kappa).all(), (rerr, kappa)
            assert terr < 1e-3, terr
        else:   # the bars of test_forward_vs_oracle_bf16; R scaled by kappa like the bf16x3 bar (B = 64 holds kappa 44)
            for k in MAPS:
                assert (out[k].cpu() - ref[k]).abs().max().item() < 0.15, k
            assert (raw[:, :6] - ref["rot6d"]).abs().max().item() < 0.06
            assert (raw[:, 6:] - ref["t_"]).abs().max().item() < 0.02
            assert (rerr < 0.1 * kappa).all(), (rerr, kappa)
            assert terr < 1e-2, terr
        del m


@pytest.mark.gpu
def test_agnostic_forward_ignores_labels(dev):
    """roi_classes=None, all-zero and arbitrary labels give identical outputs (a one-slab head reads no label), and a
    class-aware engine still refuses a NULL label pointer."""
    from gdrnpp_bop2022_b200 import _lib
    from gdrnpp_bop2022_b200.synthetic import make_batch

    m = _member(dev, 22, max_batch=8)
    gb = {k: v.to(dev) for k, v in make_batch(B=6, seed=31).items()}
    outs = [m(gb["roi_img"], **_kw(gb, roi_classes=c)) for c in
            (None, torch.zeros(6, dtype=torch.int64, device=dev), torch.tensor([3, 0, 20, 7, 1000, -5], device=dev))]
    torch.cuda.synchronize()
    for o in outs[1:]:
        for k in ("rot", "trans") + MAPS:
            assert torch.equal(o[k], outs[0][k]), k
    # the engine-level check: a 21-class head with roi_classes = NULL is an error, not class 0
    from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg
    from gdrnpp_bop2022_b200.synthetic import make_state_dict

    aware = GDRN_DoubleMask(default_cfg(), max_batch=8)
    aware.load_state_dict(make_state_dict())
    aware.to(dev)
    aware.class_aware = False       # make the Python layer pass NULL through to the C ABI
    with pytest.raises(_lib.GdrnError, match="roi_classes"):
        aware(gb["roi_img"], **_kw(gb, roi_classes=None))


@pytest.mark.gpu
def test_per_object_forward_equals_each_members_own_forward(dev):
    """Three members, 12 ROIs with shuffled labels: every ROI's rot, trans and six maps are torch.equal to its member's
    own forward over the same sub-batch in the same order -- eagerly and through the per-(member, size) graphs, twice
    each (the concurrent streams do not change a bit)."""
    from gdrnpp_bop2022_b200.per_object import PerObjectGDRN
    from gdrnpp_bop2022_b200.synthetic import make_batch

    members = {2: _member(dev, 40, max_batch=16), 5: _member(dev, 41, max_batch=16), 9: _member(dev, 42, max_batch=16)}
    labels = torch.tensor([5, 2, 9, 9, 2, 5, 5, 2, 9, 5, 2, 9])[torch.randperm(12, generator=torch.Generator().manual_seed(3))]
    gb = {k: v.to(dev) for k, v in make_batch(B=12, seed=44).items()}
    gb["roi_classes"] = labels.to(dev)
    want = {}
    for label, m in members.items():
        idx = torch.nonzero(labels == label).flatten().to(dev)
        sub = {k: v.index_select(0, idx) for k, v in gb.items()}
        o = m(sub["roi_img"], **_kw(sub, roi_classes=None))
        for k, v in o.items():
            want.setdefault(k, torch.empty((12,) + v.shape[1:], dtype=v.dtype, device=dev))[idx] = v
    torch.cuda.synchronize()
    assert set(want) == {"rot", "trans"} | set(MAPS)
    for use_graph in (False, True):
        pm = PerObjectGDRN(members, use_cuda_graph=use_graph)
        for rep in range(2):
            got = pm(gb["roi_img"], **_kw(gb))
            torch.cuda.synchronize()
            assert set(got) == set(want)
            for k in want:
                assert torch.equal(got[k], want[k]), (use_graph, rep, k)
        pm.release_graphs()
    with pytest.raises(ValueError, match=r"\[4\]"):
        PerObjectGDRN(members)(gb["roi_img"], **_kw(gb, roi_classes=torch.where(labels == 9, 4, labels)))


@pytest.mark.gpu
def test_predictor_per_object_checkpoints(dev, tmp_path):
    """GdrnPredictor with one checkpoint file per object ("_module."-prefixed keys, like the reference's saved models)
    and one per-object config: inference() returns the same poses as PerObjectGDRN over the same members on its
    data_dict, through the graph path and the eager path."""
    from gdrnpp_bop2022_b200.per_object import PerObjectGDRN
    from gdrnpp_bop2022_b200.predictor import GdrnPredictor
    from gdrnpp_bop2022_b200.synthetic import YCBV_K, make_state_dict

    objs = {1: "002_master_chef_can", 4: "005_tomato_soup_can", 7: "008_pudding_box"}
    seeds = {1: 51, 4: 52, 7: 53}
    ckpts = {}
    for oid, seed in seeds.items():
        sd = make_state_dict(num_classes=1, seed=seed)
        ckpts[oid] = str(tmp_path / f"model_{oid}.pth")
        torch.save({"model": {"_module." + k: v for k, v in sd.items()}}, ckpts[oid])
    cfg_path = _write_obj_config(tmp_path)
    extents = {1: (0.10, 0.10, 0.14), 4: (0.07, 0.07, 0.10), 7: (0.09, 0.05, 0.11)}
    rs = np.random.RandomState(8)
    image = rs.randint(0, 255, (480, 640, 3)).astype(np.uint8)
    # detections (x1, y1, x2, y2, score, cls_score, label); label = index of the object in objs
    dets = np.array([[100, 80, 220, 200, 0.9, 0.95, 2], [300, 150, 380, 260, 0.8, 0.9, 0],
                     [420, 240, 560, 400, 0.7, 0.9, 1], [50, 300, 160, 430, 0.9, 0.8, 0],
                     [250, 20, 330, 110, 0.6, 0.9, 2]], np.float32)
    for use_graph in (True, False):
        pred = GdrnPredictor(cfg_path, ckpts, cam=YCBV_K, objs=objs, extents=extents, use_pnp=False,
                             use_cuda_graph=use_graph)
        assert isinstance(pred.model, PerObjectGDRN) and sorted(pred.model.members) == [0, 1, 2]
        data = pred.preprocessing(dets, image)
        out = {k: v.clone() for k, v in pred.inference(data).items()}
        members = {}
        for label, oid in enumerate(objs):
            members[label] = _member(dev, seeds[oid], with_maps=False)
        ref = PerObjectGDRN(members)(data["roi_img"], roi_classes=data["roi_cls"], roi_coord_2d=data["roi_coord_2d"],
                                     roi_cams=data["roi_cam"], roi_centers=data["roi_center"], roi_whs=data["roi_wh"],
                                     roi_extents=data["roi_extent"], resize_ratios=data["resize_ratio"])
        torch.cuda.synchronize()
        assert torch.equal(out["rot"], ref["rot"]) and torch.equal(out["trans"], ref["trans"]), use_graph
        poses = pred.postprocessing(data, out)
        assert sorted(poses) == sorted(objs.values())
        del pred, members
