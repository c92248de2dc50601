"""Generate tests/golden/ref_heads.npz by running the REFERENCE's own Python code (imported read-only from the checkout
that GDRN_REFERENCE_SRC names) on small seeded inputs:

  * TopDownDoubleMaskXyzRegionHead   (core/gdrn_modeling/models/heads/top_down_doublemask_xyz_region_head.py)
  * ConvPnPNet                        (core/gdrn_modeling/models/heads/conv_pnp_net.py)
  * rot6d_to_mat_batch                (core/utils/rot_reps.py)
  * pose_from_predictions_test + allocentric_to_egocentric
                                      (core/gdrn_modeling/models/pose_from_pred_centroid_z.py, core/utils/utils.py)

Third-party packages the reference imports but which are absent here (mmcv, detectron2, timm, transforms3d,
numba, ...) are replaced by import stubs: a permissive dummy for everything that is only imported, and small
real implementations for the handful of functions the path executes (weight-init helpers, conv registry,
transforms3d.axangles.axangle2mat restated from its published formula).  No reference file is modified or
copied.  Reduced widths keep the fixture small (in_dim = feat_dim = 32, 3 classes, PnP featdim 32, 16x16 maps); the
weights are not stored but drawn from a seeded generator in parameter order (param_names / param_shapes), which
tests/test_oracle_pinning.py repeats.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_ref_heads.py [--agnostic]

--agnostic writes tests/golden/ref_heads_agnostic.npz instead: the class-agnostic head of the reference's per-object
models (mask / xyz / region_num_classes = 1, model_utils.py get_geo_head with the *_CLASS_AWARE flags false), same
stubs, same seeds and the same recipe, so that the channel order of a one-slab out_layer is pinned by the reference too.
"""
import importlib.abc
import importlib.machinery
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
STUB_TOPLEVEL = {"mmcv", "detectron2", "timm", "transforms3d", "numba", "fvcore", "pytorch_lightning", "loguru",
                 "termcolor", "tabulate", "imgaug", "vispy", "OpenGL", "pyassimp", "plyfile", "glumpy", "pypng", "png",
                 "ruamel", "setproctitle", "thop", "einops_exts", "open3d", "horovod", "fairscale", "tensorboardX",
                 "pycocotools", "dropblock", "iopath", "omegaconf", "hydra", "imageio", "pytz", "ipdb", "glfw",
                 "chardet", "xmltodict", "PIL_missing", "skimage", "matplotlib", "seaborn", "dill", "ujson", "lmdb"}


class Dummy:
    """Anything-goes placeholder: attribute access, calls, decorator use, iteration."""

    def __init__(self, name="dummy"):
        self.__name__ = name

    def __getattr__(self, item):
        if item.startswith("__") and item.endswith("__"):
            raise AttributeError(item)
        return Dummy(item)

    def __call__(self, *a, **k):
        if len(a) == 1 and not k and isinstance(a[0], (types.FunctionType, type)):
            return a[0]
        return self

    def __iter__(self):
        return iter(())

    def __contains__(self, item):
        return False

    def __mro_entries__(self, bases):
        return (object,)


class StubModule(types.ModuleType):
    def __getattr__(self, item):
        if item.startswith("__") and item.endswith("__"):
            raise AttributeError(item)
        return Dummy(item)


class StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    _known = {}

    def find_spec(self, fullname, path, target=None):
        top = fullname.split(".")[0]
        if top not in self._known:
            self._known[top] = top in STUB_TOPLEVEL
        if self._known[top]:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        name = module.__name__
        if name in ("mmcv.cnn", "mmcv.cnn.utils"):
            def normal_init(m, mean=0, std=1, bias=0):
                if hasattr(m, "weight") and m.weight is not None:
                    nn.init.normal_(m.weight, mean, std)
                if hasattr(m, "bias") and m.bias is not None:
                    nn.init.constant_(m.bias, bias)

            def constant_init(m, val, bias=0):
                if hasattr(m, "weight") and m.weight is not None:
                    nn.init.constant_(m.weight, val)
                if hasattr(m, "bias") and m.bias is not None:
                    nn.init.constant_(m.bias, bias)

            def kaiming_init(m, a=0, mode="fan_out", nonlinearity="relu", bias=0, distribution="normal"):
                nn.init.kaiming_normal_(m.weight, a=a, mode=mode, nonlinearity=nonlinearity)
                if hasattr(m, "bias") and m.bias is not None:
                    nn.init.constant_(m.bias, bias)

            module.normal_init, module.constant_init, module.kaiming_init = normal_init, constant_init, kaiming_init
        if name == "mmcv.cnn.bricks.conv":
            class Registry(dict):
                def register_module(self, *a, **k):
                    def deco(cls):
                        self[cls.__name__] = cls
                        return cls
                    return deco

                def get(self, k):
                    return self[k]

            reg = Registry()
            reg["Conv2d"] = nn.Conv2d
            module.CONV_LAYERS = reg
            module.build_conv_layer = lambda cfg, *a, **k: nn.Conv2d(*a, **k)
        if name == "timm.models.layers":
            class StdConv2d(nn.Conv2d):
                pass

            module.StdConv2d = StdConv2d
        if name == "detectron2.layers.batch_norm":
            module.BatchNorm2d = nn.BatchNorm2d
            module.FrozenBatchNorm2d = nn.BatchNorm2d
            module.NaiveSyncBatchNorm = nn.BatchNorm2d
        if name == "detectron2.utils":
            module.env = types.SimpleNamespace(TORCH_VERSION=(2, 0))
        if name == "detectron2.utils.env":
            module.TORCH_VERSION = (2, 0)
        if name == "detectron2.layers":
            module.cat = lambda ts, dim=0: torch.cat(ts, dim)
        if name == "transforms3d.axangles":
            def axangle2mat(axis, angle, is_normalized=False):
                x, y, z = axis
                if not is_normalized:
                    n = math.sqrt(x * x + y * y + z * z)
                    x, y, z = x / n, y / n, z / n
                c, s = math.cos(angle), math.sin(angle)
                C = 1 - c
                xs, ys, zs = x * s, y * s, z * s
                xC, yC, zC = x * C, y * C, z * C
                xyC, yzC, zxC = x * yC, y * zC, z * xC
                return np.array([[x * xC + c, xyC - zs, zxC + ys], [xyC + zs, y * yC + c, yzC - xs],
                                 [zxC - ys, yzC + xs, z * zC + c]])

            module.axangle2mat = axangle2mat


def main(agnostic=False):
    assert REF and os.path.isdir(REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    sys.meta_path.insert(0, StubFinder())
    sys.path.insert(0, REF)
    # NumPy-1.x names the reference still uses (lib/pysixd/RT_transform.py:298 etc.)
    for _n, _v in (("float", float), ("int", int), ("bool", bool), ("maximum_sctype", lambda t: np.float64)):
        if not hasattr(np, _n):
            setattr(np, _n, _v)
    torch.manual_seed(0)
    from core.gdrn_modeling.models.heads.top_down_doublemask_xyz_region_head import TopDownDoubleMaskXyzRegionHead
    from core.gdrn_modeling.models.heads.conv_pnp_net import ConvPnPNet
    from core.utils.rot_reps import rot6d_to_mat_batch
    from core.gdrn_modeling.models.pose_from_pred_centroid_z import pose_from_pred_centroid_z

    nc = 1 if agnostic else 3
    head = TopDownDoubleMaskXyzRegionHead(in_dim=32, feat_dim=32, norm="GN", num_gn_groups=32, act="GELU",
                                          mask_num_classes=nc, xyz_num_classes=nc, region_num_classes=nc,
                                          mask_out_dim=2, xyz_out_dim=3, region_out_dim=65).eval()
    pnp = ConvPnPNet(nIn=69, featdim=32, rot_dim=6, num_stride2_layers=3, norm="GN", num_gn_groups=32, act="gelu",
                     final_spatial_size=(2, 2)).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():  # non-degenerate weights (the reference init is N(0,1e-3): outputs would be ~0)
        for mod in (head, pnp):
            for n_, p in mod.named_parameters():
                if p.dim() > 1:
                    fan_in = p[0].numel() if not n_.startswith("features.0.weight") or mod is pnp else p.shape[0] * 9 / 4
                    p.copy_(torch.randn(p.shape, generator=g) * math.sqrt(2.0 / fan_in))
                elif n_.endswith("weight"):
                    p.copy_(torch.rand(p.shape, generator=g) * 0.4 + 0.8)
                else:
                    p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    B = 2
    feat = torch.randn(B, 32, 2, 2, generator=g)
    with torch.no_grad():
        vis, full, cx, cy, cz, region = head([feat])
    coor_feat = torch.rand(B, 5, 16, 16, generator=g)
    region_in = torch.softmax(torch.randn(B, 64, 16, 16, generator=g), dim=1)
    extents = torch.rand(B, 3, generator=g) * 0.2 + 0.05
    with torch.no_grad():
        rot, t = pnp(coor_feat.clone(), region=region_in, extents=extents)
    rot_m = rot6d_to_mat_batch(rot)
    cams = torch.tensor([[1066.778, 0, 312.9869], [0, 1067.487, 241.3109], [0, 0, 1]]).repeat(B, 1, 1)
    centers = torch.rand(B, 2, generator=g) * 400 + 100
    whs = torch.rand(B, 2, generator=g) * 100 + 50
    ratios = torch.rand(B, generator=g) * 0.5 + 0.3
    t_use = t.clone()
    t_use[:, 2] = t_use[:, 2].abs() + 1.0
    ego, trans = pose_from_pred_centroid_z(rot_m, pred_centroids=t_use[:, :2], pred_z_vals=t_use[:, 2:3], roi_cams=cams,
                                           roi_centers=centers, resize_ratios=ratios, roi_whs=whs, eps=1e-4,
                                           is_allo=True, z_type="REL", is_train=False)
    out = {"num_classes": np.int64(nc)}
    names, shapes, aliases, targets = [], [], [], []
    for prefix, mod in (("geo_head_net.", head), ("pnp_net.", pnp)):
        params = dict(mod.named_parameters())
        for n_, p in params.items():
            names.append(prefix + n_)
            shapes.append(",".join(str(d) for d in p.shape))
        for k, v in mod.state_dict().items():   # the same module registered twice (norm / gn): no buffers of its own
            if k not in params:
                aliases.append(prefix + k)
                targets.append(prefix + next(n_ for n_, p in params.items() if p.data_ptr() == v.data_ptr()))
    out["param_names"], out["param_shapes"] = np.array(names), np.array(shapes)
    out["alias_names"], out["alias_targets"] = np.array(aliases), np.array(targets)
    out.update({"in/feat": feat.numpy(), "in/coor_feat": coor_feat.numpy(), "in/region": region_in.numpy(),
                "in/extents": extents.numpy(), "in/cams": cams.numpy(), "in/centers": centers.numpy(),
                "in/whs": whs.numpy(), "in/ratios": ratios.numpy()})
    for name, o in zip(("vis", "full", "cx", "cy", "cz", "region"), (vis, full, cx, cy, cz, region)):
        out["out/" + name] = o.contiguous().numpy()
    out.update({"out/pnp_rot": rot.numpy(), "out/pnp_t_raw": t.numpy(), "out/pnp_t": t_use.numpy(), "out/rot_m": rot_m.numpy(),
                "out/ego_rot": ego.numpy(), "out/trans": trans.numpy()})
    path = os.path.join(ROOT, "tests", "golden", "ref_heads_agnostic.npz" if agnostic else "ref_heads.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(agnostic="--agnostic" in sys.argv[1:])
