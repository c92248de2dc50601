"""Host-side mirror of the reference model surface for the hot path.

Reference interface mirrored (paths relative to the reference tree):
  * ``build_model_optimizer(cfg, is_test)`` -> ``(model, optimizer|None)``
    (core/gdrn_modeling/models/GDRN_double_mask.py:539-615, called from main_gdrn.py:158)
  * ``GDRN_DoubleMask.forward(x, roi_classes=, roi_coord_2d=, roi_cams=, roi_centers=, roi_whs=,
    roi_extents=, resize_ratios=, do_loss=False)`` -> ``{"rot", "trans"[, "mask", "full_mask",
    "coor_x", "coor_y", "coor_z", "region"]}`` (GDRN_double_mask.py:66-214)
  * ``state_dict`` key names / shapes of a reference checkpoint (SURVEY.md Appendix A), so
    ``MyCheckpointer(model).resume_or_load`` (core/utils/my_checkpoint.py:35-83) works unchanged.

All arithmetic happens in libgdrn_b200.so (hand-written sm_90a CUDA behind the C ABI of
include/gdrn_b200.h).  There is no PyTorch/CPU fallback: without the library or a CUDA device the
forward raises.
"""
import ctypes
import os
import re
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib
from .synthetic import CONVNEXT_ARCH, state_dict_shapes


def _cfg_get(cfg, path, default=None):
    cur = cfg
    for part in path.split("."):
        if cur is None:
            return default
        if isinstance(cur, dict):
            cur = cur.get(part, None)
        else:
            cur = getattr(cur, part, None)
    return default if cur is None else cur


def default_cfg(num_classes=21, arch="convnext_base", with_maps=False):
    """Minimal stand-in for the mmcv Config of convnext_a6_AugCosyAAEGray_..._ycbv.py (SURVEY.md Appendix A)."""
    return SimpleNamespace(
        MODEL=SimpleNamespace(
            POSE_NET=SimpleNamespace(
                NAME="GDRN_double_mask",
                NUM_CLASSES=num_classes,
                OUTPUT_RES=64,
                BACKBONE=SimpleNamespace(INIT_CFG=SimpleNamespace(type="timm/" + arch)),
                GEO_HEAD=SimpleNamespace(NUM_REGIONS=64, XYZ_CLASS_AWARE=True, MASK_CLASS_AWARE=True,
                                         REGION_CLASS_AWARE=True),
                PNP_NET=SimpleNamespace(ROT_TYPE="allo_rot6d", TRANS_TYPE="centroid_z", Z_TYPE="REL",
                                        WITH_2D_COORD=True, REGION_ATTENTION=True),
            )
        ),
        TEST=SimpleNamespace(USE_PNP=with_maps, SAVE_RESULTS_ONLY=False, USE_DEPTH_REFINE=with_maps),
        INPUT=SimpleNamespace(WITH_DEPTH=False),
    )


class _NS(SimpleNamespace):
    """Attribute + item access, like the mmcv ConfigDict the reference passes around."""

    def __getitem__(self, k):
        return getattr(self, k)

    def get(self, k, default=None):
        return getattr(self, k, default)


def _to_ns(d):
    if isinstance(d, dict):
        return _NS(**{k: _to_ns(v) for k, v in d.items()})
    return d


def _merge(base, new):
    out = dict(base)
    for k, v in new.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict) and not v.get("_delete_", False):
            out[k] = _merge(out[k], v)
        else:
            out[k] = {kk: vv for kk, vv in v.items() if kk != "_delete_"} if isinstance(v, dict) else v
    return out


def load_py_config(path):
    """Read a reference-style python config (configs/gdrn/**.py: module-level dicts, ``_base_`` inheritance with key-wise
    dict merge like mmcv.Config.fromfile) into a nested attribute namespace.  Only the few fields the hot path reads
    are interpreted (MODEL.POSE_NET.*, TEST.*, INPUT.*); the rest of the reference's config system is out of scope."""
    import os as _os

    def _load(p):
        scope = {}
        with open(p) as f:
            exec(compile(f.read(), p, "exec"), scope)   # noqa: S102  (configs are python files in the reference too)
        cur = {k: v for k, v in scope.items() if not k.startswith("__") and isinstance(v, (dict, list, tuple, str, int, float, bool, type(None)))}
        bases = cur.pop("_base_", [])
        if isinstance(bases, str):
            bases = [bases]
        merged = {}
        for b in bases:
            merged = _merge(merged, _load(_os.path.join(_os.path.dirname(p), b)))
        return _merge(merged, cur)

    return _to_ns(_load(path))


class _Shell(nn.Module):
    """Parameter container reproducing the reference module tree (no forward of its own)."""


def _build_param_tree(root, shapes):
    for key, shape in shapes.items():
        parts = key.split(".")
        mod = root
        for p in parts[:-1]:
            if p not in mod._modules:
                mod.add_module(p, _Shell())
            mod = mod._modules[p]
        mod.register_parameter(parts[-1], nn.Parameter(torch.zeros(shape), requires_grad=False))


class GDRN_DoubleMask(nn.Module):
    def __init__(self, cfg, arch="convnext_base", max_batch=64, precision=None):
        """precision: "bf16x3" (default; split-bf16 tensor-core GEMMs that reproduce the reference's fp32 forward: R within
        1e-4 rad / t within 1e-3, the mode every headline number is quoted in) or "bf16" (single bf16 operands, ~2x the
        throughput, R within ~0.03 rad: the regime of the reference's AMP test path; see include/gdrn_b200.h).
        None -> cfg.MODEL.POSE_NET.PRECISION if present, else the GDRN_PRECISION environment variable (0 = bf16,
        1 = bf16x3), else bf16x3."""
        super().__init__()
        net_cfg = cfg.MODEL.POSE_NET
        assert net_cfg.NAME == "GDRN_double_mask", net_cfg.NAME
        self.cfg = cfg
        self.arch = arch
        self.num_classes = int(net_cfg.NUM_CLASSES)
        self.max_batch = max_batch
        if precision is None:
            precision = getattr(net_cfg, "PRECISION", None)
        if precision is None:
            precision = {"0": "bf16", "1": "bf16x3"}.get(os.environ.get("GDRN_PRECISION", "1"), "bf16x3")
        if precision not in ("bf16", "bf16x3"):
            raise ValueError(f"precision must be 'bf16' or 'bf16x3', got {precision!r}")
        self.precision = precision
        self.neck = None
        if arch not in CONVNEXT_ARCH:
            raise ValueError(f"unknown backbone {arch}")
        pnp = net_cfg.PNP_NET
        if pnp.ROT_TYPE != "allo_rot6d" or pnp.TRANS_TYPE != "centroid_z" or _cfg_get(pnp, "Z_TYPE", "REL") != "REL":
            raise NotImplementedError("this path implements ROT_TYPE=allo_rot6d, TRANS_TYPE=centroid_z, Z_TYPE=REL")
        g = net_cfg.GEO_HEAD
        aware = (bool(g.XYZ_CLASS_AWARE), bool(g.MASK_CLASS_AWARE), bool(g.REGION_CLASS_AWARE))
        if len(set(aware)) != 1 or g.NUM_REGIONS != 64:
            raise NotImplementedError("this path implements the 64-region geometry head, either class-aware or "
                                      "class-agnostic in all of xyz / mask / region")
        # class-agnostic (the reference's per-object models, model_utils.get_geo_head): one class slab of 70 channels,
        # the class gather is skipped and roi_classes is not read
        self.class_aware = aware[0]
        self.head_classes = self.num_classes if self.class_aware else 1
        shapes = state_dict_shapes(arch, self.head_classes)
        _build_param_tree(self, shapes)
        self._handle = None
        self._engine_device = None   # the CUDA device the engine's weights live on (cudaMalloc'ed on first use)
        self._loaded_version = None
        self._workspace = None
        self._graph_pinned = False   # a captured CUDA graph holds raw workspace / weight pointers
        self._param_version = 0

    # --- weights ---------------------------------------------------------------------------------
    def _load_from_state_dict(self, *args, **kwargs):
        self._param_version += 1
        return super()._load_from_state_dict(*args, **kwargs)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._param_version += 1
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def mark_weights_dirty(self):
        self._param_version += 1

    def _ensure_engine(self, device):
        """Create the engine on ``device`` (made current by the caller) and (re)load dirty weights.  The engine is
        bound to the device it was created on: weights are cudaMalloc'ed there and the kernels' shared-memory opt-in is
        per device, so a later forward on another device raises instead of silently running on the wrong GPU."""
        L = _lib.lib()
        if self._engine_device is not None and self._engine_device != device:
            raise _lib.GdrnError(f"this model's engine lives on {self._engine_device}; got tensors on {device} "
                                 "(build one GDRN_DoubleMask per device)")
        if self._handle is None:
            h = ctypes.c_void_p()
            _lib.check(L.gdrn_model_create_ex(ctypes.byref(h), self.arch.encode(), self.head_classes, self.max_batch,
                                              1 if self.precision == "bf16x3" else 0), "gdrn_model_create_ex")
            self._handle = h
            self._engine_device = device
        if self._loaded_version != self._param_version:
            if self._graph_pinned:
                raise _lib.GdrnError("weights changed after capture_graph(): the captured graph does not re-run the "
                                     "weight re-pack; re-capture (model.release_graphs()) before reloading weights")
            st = _lib.current_stream()
            for k, v in self.state_dict().items():
                t = v.detach().to(device=device, dtype=torch.float32).contiguous()
                _lib.check(L.gdrn_model_load_tensor(self._handle, k.encode(), _lib.ptr(t), t.numel(), st),
                           f"gdrn_model_load_tensor({k})")
            torch.cuda.current_stream().synchronize()  # sources may be temporaries
            missing = L.gdrn_model_missing(self._handle)
            if missing != 0:
                raise _lib.GdrnError(f"{missing} weight tensors missing after load")
            self._loaded_version = self._param_version

    def _get_workspace(self, B, device):
        need = _lib.lib().gdrn_model_workspace_bytes(self._handle, B)
        if self._workspace is None or self._workspace.numel() < need or self._workspace.device != device:
            self._workspace = torch.empty(need, dtype=torch.uint8, device=device)
        return self._workspace

    def release_graphs(self):
        """Forget that CUDA graphs were captured from this model (the caller drops its replay closures)."""
        self._graph_pinned = False

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.lib().gdrn_model_destroy(self._handle)
        except Exception:
            pass

    @property
    def wants_maps(self):
        """True when the config asks for the geometry maps (PnP, result saving or depth refine read them)."""
        cfg = self.cfg
        return bool(_cfg_get(cfg, "TEST.USE_PNP", False) or _cfg_get(cfg, "TEST.SAVE_RESULTS_ONLY", False)
                    or _cfg_get(cfg, "TEST.USE_DEPTH_REFINE", False))

    # --- forward ---------------------------------------------------------------------------------
    def forward(self, x, gt_xyz=None, gt_xyz_bin=None, gt_mask_trunc=None, gt_mask_visib=None, gt_mask_obj=None,
                gt_mask_full=None, gt_region=None, gt_ego_rot=None, gt_points=None, sym_infos=None, gt_trans=None,
                gt_trans_ratio=None, roi_classes=None, roi_coord_2d=None, roi_coord_2d_rel=None, roi_cams=None,
                roi_centers=None, roi_whs=None, roi_extents=None, resize_ratios=None, do_loss=False,
                return_raw=False, _workspace=None):
        if do_loss:
            raise NotImplementedError("training (do_loss=True) is out of scope of the inference hot path")
        if not x.is_cuda:
            raise _lib.GdrnError("GDRN_DoubleMask.forward needs CUDA tensors (no CPU fallback)")
        for name, t in (("roi_classes", roi_classes if self.class_aware else 0), ("roi_coord_2d", roi_coord_2d),
                        ("roi_cams", roi_cams), ("roi_centers", roi_centers), ("roi_whs", roi_whs),
                        ("roi_extents", roi_extents), ("resize_ratios", resize_ratios)):
            if t is None:
                raise ValueError(f"{name} is required")
        dev = x.device
        B = x.shape[0]
        if tuple(x.shape[1:]) != (3, 256, 256):
            raise ValueError(f"roi_img must be [B,3,256,256], got {tuple(x.shape)}")
        want_maps = self.wants_maps
        map_names = (("mask", 1), ("full_mask", 1), ("coor_x", 1), ("coor_y", 1), ("coor_z", 1), ("region", 65))
        out_rot = torch.empty((B, 3, 3), dtype=torch.float32, device=dev)
        out_trans = torch.empty((B, 3), dtype=torch.float32, device=dev)
        out_raw = torch.empty((B, 9), dtype=torch.float32, device=dev) if return_raw else None
        tensors = {}
        if want_maps:
            for name, ch in map_names:
                tensors[name] = torch.empty((B, ch, 64, 64), dtype=torch.float32, device=dev)
        out = {"rot": out_rot, "trans": out_trans}
        out.update(tensors)
        if return_raw:
            out["raw"] = out_raw
        if B == 0:   # the reference forward is shape-polymorphic in B; an image without detections yields empty poses
            return out
        with torch.cuda.device(dev):   # the C ABI works on the CURRENT device / its current stream
            self._ensure_engine(dev)
            f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
            x = f32(x)
            # class-agnostic head: the labels are not read (GDRN_double_mask.py skips the class gathers), NULL to the engine
            cls = roi_classes.detach().to(device=dev, dtype=torch.int64).contiguous() if self.class_aware else None
            if roi_cams.dim() == 2:
                roi_cams = roi_cams.unsqueeze(0).expand(B, 3, 3)
            c2d, cams, ctr, whs, ext, rr = (f32(roi_coord_2d), f32(roi_cams), f32(roi_centers), f32(roi_whs),
                                            f32(roi_extents), f32(resize_ratios.reshape(-1)))
            L = _lib.lib()
            # more ROIs than the engine's max_batch: run contiguous chunks (the reference has no batch limit)
            for b0 in range(0, B, self.max_batch):
                n = min(self.max_batch, B - b0)
                sl = slice(b0, b0 + n)
                maps = None
                if want_maps:
                    maps = _lib.GdrnMaps(*[tensors[nm][sl].data_ptr() for nm, _ in map_names])
                ws = _workspace if _workspace is not None else self._get_workspace(n, dev)
                rc = L.gdrn_model_forward(
                    self._handle, _lib.ptr(x[sl]), _lib.ptr(cls[sl]) if cls is not None else None, _lib.ptr(c2d[sl]),
                    _lib.ptr(cams[sl]),
                    _lib.ptr(ctr[sl]), _lib.ptr(whs[sl]), _lib.ptr(rr[sl]), _lib.ptr(ext[sl]), n, _lib.ptr(out_rot[sl]),
                    _lib.ptr(out_trans[sl]), _lib.ptr(out_raw[sl]) if out_raw is not None else None,
                    ctypes.byref(maps) if maps is not None else None, _lib.ptr(ws), ws.numel(), _lib.current_stream())
                _lib.check(rc, "gdrn_model_forward")
        return out

    def capture_graph(self, batch, warmup=2):
        """Capture one forward over the STATIC tensors of ``batch`` (reference data_dict keys: roi_img, roi_classes,
        roi_coord_2d, roi_cams, roi_centers, roi_whs, roi_extents, resize_ratios) into a CUDA graph.

        Returns ``(replay, out_dict)``: ``replay()`` re-runs the ~150 kernel launches of the forward as one graph
        launch on the current stream (inputs are read from the same tensors, so refill them in place);
        ``out_dict`` holds the static output tensors.  CUDA streams and graphs replace a tracing compiler here.
        A class-agnostic model does not read roi_classes, which may then be absent or None."""
        kw = dict(roi_classes=batch["roi_classes"] if self.class_aware else None, roi_coord_2d=batch["roi_coord_2d"],
                  roi_cams=batch["roi_cams"], roi_centers=batch["roi_centers"], roi_whs=batch["roi_whs"],
                  roi_extents=batch["roi_extents"], resize_ratios=batch["resize_ratios"])
        for k, v in list(kw.items()) + [("roi_img", batch["roi_img"])]:
            if k == "roi_classes" and not self.class_aware:
                continue
            if not (v is not None and v.is_cuda and v.is_contiguous()):
                raise _lib.GdrnError(f"capture_graph: {k} must be a contiguous CUDA tensor")
        if batch["roi_img"].dtype != torch.float32 or (self.class_aware and batch["roi_classes"].dtype != torch.int64):
            raise _lib.GdrnError("capture_graph: roi_img must be float32 and roi_classes int64 (no hidden copies)")
        dev = batch["roi_img"].device
        B = batch["roi_img"].shape[0]
        if B < 1 or B > self.max_batch:
            raise _lib.GdrnError(f"capture_graph: batch {B} outside [1, max_batch={self.max_batch}]")
        with torch.cuda.device(dev):
            self._ensure_engine(dev)
            # The graph bakes raw pointers in: give it its OWN workspace (kept alive by the returned closure) instead
            # of self._workspace, which later eager forwards may re-allocate.
            ws = torch.empty(_lib.lib().gdrn_model_workspace_bytes(self._handle, B), dtype=torch.uint8, device=dev)
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(warmup):
                    self.forward(batch["roi_img"], _workspace=ws, **kw)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self.forward(batch["roi_img"], _workspace=ws, **kw)
        self._graph_pinned = True

        def replay(_graph=graph, _ws=ws):
            _graph.replay()

        return replay, out

    def debug_read(self, name, B, numel):
        dst = torch.empty(numel, dtype=torch.float32, device=self._workspace.device)
        n = _lib.lib().gdrn_model_debug_read(self._handle, name.encode(), B, _lib.ptr(dst), _lib.ptr(self._workspace),
                                             _lib.current_stream())
        if n < 0:
            raise _lib.GdrnError(f"debug_read({name}) failed: {_lib.last_error()}")
        return dst[:n]

    def run_stage(self, stage, x, roi_classes=None, roi_extents=None, roi_coord_2d=None, want_raw=False, want_maps=False):
        """One backbone / geometry-head / Patch-PnP stage of the forward on the fp32 CUDA tensor ``x`` (NCHW roi_img for
        "stem", NHWC otherwise; gdrn_model_run_stage in include/gdrn_b200.h lists the stages and shapes).  Returns
        ``{"out"}`` plus, when ``want_raw``, ``"raw"`` (head stages: the conv output before GroupNorm; "down<s>" /
        "block<s>_<i>": the GEMM operand written by the LayerNorm kernel) and, for the head stages, ``"gn_stats"`` (float64
        [10,B,32,2]), and, when ``want_maps``, the six NCHW maps of "out_conv"."""
        dev = x.device
        B = x.shape[0]
        x = x.detach().to(dtype=torch.float32).contiguous()
        depths, dims = CONVNEXT_ARCH[self.arch]
        cp = [(d + 63) // 64 * 64 for d in dims]   # stored stage widths (zero pad channels)
        m_down = re.fullmatch(r"down([1-3])", stage)
        m_block = re.fullmatch(r"block([0-3])_(0|[1-9][0-9]*)", stage)
        gn = False
        if stage == "stem":
            out_shape, raw_shape = (B, 64, 64, cp[0]), None
        elif m_down:
            s = int(m_down.group(1))
            r = 64 >> s
            out_shape, raw_shape = (B, r, r, cp[s]), (B, r, r, 4 * cp[s - 1])
        elif m_block and int(m_block.group(2)) < depths[int(m_block.group(1))]:
            s = int(m_block.group(1))
            r = 64 >> s
            out_shape = raw_shape = (B, r, r, cp[s])
        elif stage == "deconv":
            out_shape, raw_shape, gn = (B, 16, 16, 256), (B, 16, 16, 256), True
        elif re.fullmatch(r"head_conv[0-5]", stage):
            li = int(stage[len("head_conv"):])
            h = 16 << (li // 2)
            ho = 2 * h if li in (1, 3) else h
            out_shape, raw_shape, gn = (B, ho, ho, 256), (B, h, h, 256), True
        elif stage == "out_conv":
            out_shape, raw_shape = (B, 64, 64, 128), None
        elif re.fullmatch(r"pnp_conv[0-2]", stage):
            r = 32 >> int(stage[len("pnp_conv"):])
            out_shape, raw_shape, gn = (B, r, r, 128), (B, r, r, 128), True
        elif stage == "pnp_fc":
            out_shape, raw_shape = (B, 16), None
        else:
            raise ValueError(f"unknown stage {stage!r} for {self.arch}")
        res = {"out": torch.empty(out_shape, dtype=torch.float32, device=dev)}
        if want_raw:
            if raw_shape is None:
                raise ValueError(f"stage {stage!r} has no conv output / operand to return")
            res["raw"] = torch.empty(raw_shape, dtype=torch.float32, device=dev)
            if gn:
                res["gn_stats"] = torch.empty((10, B, 32, 2), dtype=torch.float64, device=dev)
        maps = None
        if want_maps:
            for name, ch in (("mask", 1), ("full_mask", 1), ("coor_x", 1), ("coor_y", 1), ("coor_z", 1), ("region", 65)):
                res[name] = torch.empty((B, ch, 64, 64), dtype=torch.float32, device=dev)
            maps = _lib.GdrnMaps(*[res[k].data_ptr() for k in ("mask", "full_mask", "coor_x", "coor_y", "coor_z", "region")])
        f32 = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float32).contiguous()
        cls = None if roi_classes is None else roi_classes.detach().to(device=dev, dtype=torch.int64).contiguous()
        ext, c2d = f32(roi_extents), f32(roi_coord_2d)
        with torch.cuda.device(dev):
            self._ensure_engine(dev)
            ws = self._get_workspace(B, dev)
            rc = _lib.lib().gdrn_model_run_stage(
                self._handle, stage.encode(), B, _lib.ptr(x), _lib.ptr(res["out"]), _lib.ptr(res.get("raw")),
                _lib.ptr(res.get("gn_stats")), _lib.ptr(cls), _lib.ptr(ext), _lib.ptr(c2d),
                ctypes.byref(maps) if maps is not None else None, _lib.ptr(ws), ws.numel(), _lib.current_stream())
            _lib.check(rc, f"gdrn_model_run_stage({stage})")
        return res


def build_model_optimizer(cfg, is_test=True):
    """Reference entry point (GDRN_double_mask.py:539-615).  Only the test-time build is in scope."""
    if not is_test:
        raise NotImplementedError("training is out of scope of the inference hot path (SURVEY.md §2 row 17/19)")
    bb_type = _cfg_get(cfg, "MODEL.POSE_NET.BACKBONE.INIT_CFG.type", "timm/convnext_base")
    arch = bb_type.split("/")[-1]
    model = GDRN_DoubleMask(cfg, arch=arch)
    return model, None
