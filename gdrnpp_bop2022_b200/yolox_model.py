"""The YOLOX detector network (det/yolox/models: YOLOX(YOLOPAFPN(depth, width), YOLOXHead(num_classes, width))) on the
CUDA kernels of csrc/yolox_net.cu, and a reader of the reference's YOLOX LazyConfig files.

``YOLOX`` carries the reference's state-dict keys (``backbone.backbone.stem.conv.conv.weight``, ``...bn.running_var``,
``num_batches_tracked``, ``head.cls_preds.0.bias``, ...), unfused or fused (conv bias, no ``bn``: what fuse_model saves).
Its forward returns ``{"det_preds": [B, A, 5 + nc]}`` decoded like ``YOLOXHead`` with ``decode_in_inference=True``.

At the first forward for an input size the state dict goes to the C ABI engine of csrc/yolox_net.cu (yolox_model_*),
which folds the BatchNorms into the conv weights in float64 (fuse_conv_and_bn, det/yolox/utils/model_utils.py:33-58,
eps 1e-3 as YOLOX.init_yolo sets it), packs them for the implicit-GEMM conv kernel and lays the layer plan out over fp32
NHWC activation buffers in a workspace the module owns (the C caller owns it).  Concatenations are channel slices of
those buffers: every producer writes its slice directly, so torch.cat costs nothing.  The two first head 3x3 convs of a
level (cls_convs[k][0], reg_convs[k][0]) read the same stem output and run as one conv with doubled N; reg + obj
predictions are one conv over reg_feat and the class predictions one over cls_feat, both into one raw buffer per level.
A forward is 156 launches at YOLOX-X; ``capture_graph`` replays them as one CUDA graph.  No CPU fallback.

``forward(x, augment=True, cfg=cfg)`` is the reference's multi-scale test-time augmentation (det/yolox/models/yolox.py:53-86,
what ``test.augment = True`` / ``test.scales`` select): for each scale s of ``cfg.scales`` the input is resampled like
model_utils.scale_img (bilinear to int(H*s) x int(W*s), padded with 0.447*255 to a multiple of 32), run through the
network, its boxes divided by s, and the outputs concatenated along the anchor axis in scale order.  The same engine
serves every scale: one layer plan per input size over one set of packed weights.  The resampling happens inside the
Focus kernel of each scaled plan, so the scaled images are never stored.
"""
import ast
import ctypes
import os
from collections.abc import Mapping
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib

BN_EPS = 1e-3
STRIDES = (8, 16, 32)


# ---------------------------------------------------------------------------------------------------------------------
# module tree with the reference's names (det/yolox/models/network_blocks.py, darknet.py, yolo_pafpn.py, yolo_head.py)
# ---------------------------------------------------------------------------------------------------------------------
class BaseConv(nn.Module):
    def __init__(self, cin, cout, ksize, stride=1):
        super().__init__()
        self.stride = stride
        self.conv = nn.Conv2d(cin, cout, ksize, stride, (ksize - 1) // 2, bias=False)
        self.bn = nn.BatchNorm2d(cout, eps=BN_EPS, momentum=0.03)

    def to_fused_layout(self):
        if self.bn is not None:
            self.conv.bias = nn.Parameter(torch.zeros(self.conv.out_channels, device=self.conv.weight.device))
            self.bn = None

    def folded(self):
        """(W [Cout, Cin, k, k], b [Cout]) float64 with the BatchNorm folded in (fuse_conv_and_bn)."""
        w = self.conv.weight.detach().double().cpu()
        cb = None if self.conv.bias is None else self.conv.bias.detach().double().cpu()
        if self.bn is None:
            return w, (torch.zeros(w.shape[0], dtype=torch.float64) if cb is None else cb)
        return fold_bn(w, self.bn.weight.detach().double().cpu(), self.bn.bias.detach().double().cpu(),
                       self.bn.running_mean.double().cpu(), self.bn.running_var.double().cpu(), cb, self.bn.eps)


def fold_bn(w, bn_w, bn_b, mean, var, conv_bias=None, eps=BN_EPS):
    """fuse_conv_and_bn (det/yolox/utils/model_utils.py:33-58) in the dtype of the inputs."""
    w_bn = torch.diag(bn_w.div(torch.sqrt(eps + var)))
    fw = torch.mm(w_bn, w.reshape(w.shape[0], -1)).view(w.shape)
    b_conv = torch.zeros(w.shape[0], dtype=w.dtype) if conv_bias is None else conv_bias
    b_bn = bn_b - bn_w.mul(mean).div(torch.sqrt(var + eps))
    return fw, torch.mm(w_bn, b_conv.reshape(-1, 1)).reshape(-1) + b_bn


class Bottleneck(nn.Module):
    def __init__(self, c, shortcut):
        super().__init__()
        self.conv1 = BaseConv(c, c, 1)
        self.conv2 = BaseConv(c, c, 3)
        self.use_add = shortcut


class CSPLayer(nn.Module):
    def __init__(self, cin, cout, n, shortcut=True):
        super().__init__()
        h = int(cout * 0.5)
        self.hidden = h
        self.conv1 = BaseConv(cin, h, 1)
        self.conv2 = BaseConv(cin, h, 1)
        self.conv3 = BaseConv(2 * h, cout, 1)
        self.m = nn.Sequential(*[Bottleneck(h, shortcut) for _ in range(n)])


class Focus(nn.Module):
    def __init__(self, cout):
        super().__init__()
        self.conv = BaseConv(12, cout, 3)


class SPPBottleneck(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        h = cin // 2
        self.conv1 = BaseConv(cin, h, 1)
        self.conv2 = BaseConv(4 * h, cout, 1)


class CSPDarknet(nn.Module):
    def __init__(self, depth, width):
        super().__init__()
        b = int(width * 64)
        bd = max(round(depth * 3), 1)
        self.stem = Focus(b)
        self.dark2 = nn.Sequential(BaseConv(b, 2 * b, 3, 2), CSPLayer(2 * b, 2 * b, bd))
        self.dark3 = nn.Sequential(BaseConv(2 * b, 4 * b, 3, 2), CSPLayer(4 * b, 4 * b, 3 * bd))
        self.dark4 = nn.Sequential(BaseConv(4 * b, 8 * b, 3, 2), CSPLayer(8 * b, 8 * b, 3 * bd))
        self.dark5 = nn.Sequential(BaseConv(8 * b, 16 * b, 3, 2), SPPBottleneck(16 * b, 16 * b),
                                   CSPLayer(16 * b, 16 * b, bd, shortcut=False))


class YOLOPAFPN(nn.Module):
    def __init__(self, depth, width, in_channels=(256, 512, 1024)):
        super().__init__()
        c0, c1, c2 = (int(c * width) for c in in_channels)
        n = round(3 * depth)
        self.backbone = CSPDarknet(depth, width)
        self.lateral_conv0 = BaseConv(c2, c1, 1)
        self.C3_p4 = CSPLayer(2 * c1, c1, n, False)
        self.reduce_conv1 = BaseConv(c1, c0, 1)
        self.C3_p3 = CSPLayer(2 * c0, c0, n, False)
        self.bu_conv2 = BaseConv(c0, c0, 3, 2)
        self.C3_n3 = CSPLayer(2 * c0, c1, n, False)
        self.bu_conv1 = BaseConv(c1, c1, 3, 2)
        self.C3_n4 = CSPLayer(2 * c1, c2, n, False)


class YOLOXHead(nn.Module):
    def __init__(self, num_classes, width, in_channels=(256, 512, 1024)):
        super().__init__()
        ch = int(256 * width)
        self.num_classes = num_classes
        # registration order of the reference (state-dict key order)
        self.cls_convs = nn.ModuleList(nn.Sequential(BaseConv(ch, ch, 3), BaseConv(ch, ch, 3)) for _ in in_channels)
        self.reg_convs = nn.ModuleList(nn.Sequential(BaseConv(ch, ch, 3), BaseConv(ch, ch, 3)) for _ in in_channels)
        self.cls_preds = nn.ModuleList(nn.Conv2d(ch, num_classes, 1) for _ in in_channels)
        self.reg_preds = nn.ModuleList(nn.Conv2d(ch, 4, 1) for _ in in_channels)
        self.obj_preds = nn.ModuleList(nn.Conv2d(ch, 1, 1) for _ in in_channels)
        self.stems = nn.ModuleList(BaseConv(int(c * width), ch, 1) for c in in_channels)


def _base_convs(module):
    return [m for m in module.modules() if isinstance(m, BaseConv)]


# ---------------------------------------------------------------------------------------------------------------------
# engine: the C ABI model of csrc/yolox_net.cu for one (device, max_batch, H, W, precision)
# ---------------------------------------------------------------------------------------------------------------------
class _Engine:
    def __init__(self, model, device, H, W, load=True):
        """``load=False`` leaves the weights out: such an engine only lays plans out (host only, no device call), for
        the step-table entries below."""
        L = _lib.lib()
        self.device = device
        h = ctypes.c_void_p()
        _lib.check(L.yolox_model_create(ctypes.byref(h), model.depth, model.width, model.num_classes, model.max_batch, H, W,
                                         1 if model.precision == "bf16x3" else 0), "yolox_model_create")
        self.handle = h
        self.A = L.yolox_model_num_anchors(h)
        self.scales, self.A_tta = None, 0   # the test-time-augmentation scale set (yolox_model_set_scales)
        self.workspace = None
        if not load:
            return
        st = _lib.current_stream()
        for k, v in model.state_dict().items():
            if k.endswith("num_batches_tracked"):
                continue
            t = v.detach().to(device=device, dtype=torch.float32).contiguous()
            _lib.check(L.yolox_model_load_tensor(h, k.encode(), _lib.ptr(t), t.numel(), st), f"yolox_model_load_tensor({k})")
        missing = L.yolox_model_missing(h)
        if missing != 0:
            raise _lib.GdrnError(f"yolox_model_missing: {missing} convs lack a tensor ({_lib.last_error()})")

    def set_scales(self, scales):
        """Lay out one plan per scale (host only); a no-op when the set is unchanged."""
        if scales != self.scales:
            L = _lib.lib()
            _lib.check(L.yolox_model_set_scales(self.handle, (ctypes.c_double * len(scales))(*scales), len(scales)),
                       "yolox_model_set_scales")
            self.scales, self.A_tta = scales, L.yolox_model_num_anchors_tta(self.handle)

    def workspace_bytes(self, B, tta=False):
        L = _lib.lib()
        return (L.yolox_model_workspace_bytes_tta if tta else L.yolox_model_workspace_bytes)(self.handle, B)

    def new_workspace(self, B, tta=False):
        return torch.empty(self.workspace_bytes(B, tta), dtype=torch.uint8, device=self.device)

    def run(self, x, det, ws, tta=False):
        fn, name = (_lib.lib().yolox_model_forward_tta, "yolox_model_forward_tta") if tta else (_lib.lib().yolox_model_forward,
                                                                                              "yolox_model_forward")
        _lib.check(fn(self.handle, _lib.ptr(x), x.shape[0], _lib.ptr(det), _lib.ptr(ws), ws.numel(), _lib.current_stream()), name)

    # -- test / measurement entries (yolox_model_plan_info / step_info / buffer_info / run_step in include/gdrn_b200.h) --
    STEP_KINDS = ("conv", "focus", "spp", "upsample", "head")
    STEP_SLOTS = ("kind", "src", "s_off", "s_c", "dst", "d_off", "d_c", "res", "r_off", "in_h", "in_w", "out_h", "out_w", "ks",
                  "stride", "act", "level_stride", "anchor_off")

    def plan_info(self, plan=0):
        """-> dict(n_steps, n_bufs, H, W, sh, sw, A, A_row, a_base) of plan ``plan`` (0: the create-time size; 1..: the
        non-unit scales of the current scale set)."""
        info = (ctypes.c_int * 9)()
        _lib.check(_lib.lib().yolox_model_plan_info(self.handle, plan, info), "yolox_model_plan_info")
        return dict(zip(("n_steps", "n_bufs", "H", "W", "sh", "sw", "A", "A_row", "a_base"), info))

    def steps(self, plan=0):
        """The step table of a plan: one dict per step with the slots of yolox_model_step_info, ``kind`` as a name and
        ``name`` the packed conv name ("" for other kinds)."""
        out = []
        info, name = (ctypes.c_int * len(self.STEP_SLOTS))(), ctypes.create_string_buffer(256)
        for i in range(self.plan_info(plan)["n_steps"]):
            _lib.check(_lib.lib().yolox_model_step_info(self.handle, plan, i, info, name, 256), "yolox_model_step_info")
            d = dict(zip(self.STEP_SLOTS, info))
            d["kind"], d["name"] = self.STEP_KINDS[d["kind"]], name.value.decode()
            out.append(d)
        return out

    def buffer_info(self, plan, buf, batch):
        """-> (byte offset from the 256-aligned workspace base, pixels per image, ld, workspace bytes the plan needs) of
        buffer ``buf`` of a plan laid out for ``batch`` images."""
        info = (ctypes.c_int64 * 4)()
        _lib.check(_lib.lib().yolox_model_buffer_info(self.handle, plan, buf, batch, info), "yolox_model_buffer_info")
        return tuple(info)

    def buffer(self, ws, plan, buf, batch):
        """The fp32 view [batch, pixels, ld] of buffer ``buf`` of a plan laid out for ``batch`` images inside the uint8
        workspace tensor ``ws``."""
        off, pix, ld, need = self.buffer_info(plan, buf, batch)
        if ws.numel() < need:
            raise _lib.GdrnError(f"workspace of {ws.numel()} bytes, plan {plan} needs {need} at batch {batch}")
        start = (-ws.data_ptr()) % 256 + off
        return ws[start:start + batch * pix * ld * 4].view(torch.float32).view(batch, pix, ld)

    def run_step(self, x, det, ws, plan, step):
        """Run step ``step`` of ``plan`` for the x.shape[0] <= max_batch images of x, writing det's rows as the forward
        (plan 0) or the TTA forward (plan >= 1) does."""
        _lib.check(_lib.lib().yolox_model_run_step(self.handle, plan, step, _lib.ptr(x), x.shape[0], _lib.ptr(det), _lib.ptr(ws),
                                                   ws.numel(), _lib.current_stream()), "yolox_model_run_step")

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().yolox_model_destroy(self.handle)
        except Exception:  # noqa: BLE001 -- interpreter shutdown
            pass


class YOLOX(nn.Module):
    """YOLOX(YOLOPAFPN(depth, width), YOLOXHead(num_classes, width)) for inference on the GPU.  precision "bf16x3"
    (split-bf16 operands, the default) or "bf16"; batches larger than ``max_batch`` run in chunks."""

    def __init__(self, depth=1.33, width=1.25, num_classes=80, max_batch=8, precision="bf16x3"):
        super().__init__()
        if precision not in ("bf16x3", "bf16"):
            raise ValueError(f"precision must be 'bf16x3' or 'bf16', got {precision!r}")
        self.depth, self.width, self.num_classes = float(depth), float(width), int(num_classes)
        self.max_batch, self.precision = int(max_batch), precision
        self.c_in = tuple(int(c * width) for c in (256, 512, 1024))
        self.backbone = YOLOPAFPN(depth, width)
        self.head = YOLOXHead(num_classes, width)
        self._engines = {}
        self._param_version = 0
        self._graph_pinned = False

    def fuse(self):
        """Replace every conv + BatchNorm by the folded conv (fuse_model): the state dict then has conv biases and no bn."""
        with torch.no_grad():
            for m in _base_convs(self):
                if m.bn is not None:
                    w, b = m.folded()
                    m.conv.weight.copy_(w.to(m.conv.weight))
                    m.to_fused_layout()
                    m.conv.bias.copy_(b.to(m.conv.bias))
        self._param_version += 1
        return self

    def load_state_dict(self, state_dict, strict=True, **kw):
        fused = not any(".bn." in k for k in state_dict) and any(k.endswith("stem.conv.conv.bias") for k in state_dict)
        if fused:
            for m in _base_convs(self):
                m.to_fused_layout()
        self._param_version += 1
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _engine(self, device, H, W):
        if self._engines and next(iter(self._engines.values())).device != device:
            raise _lib.GdrnError("this YOLOX's engine lives on another device; build one model per device")
        key = (H, W)
        eng = self._engines.get(key)
        if eng is not None and eng.version != self._param_version:
            if self._graph_pinned:
                raise _lib.GdrnError("weights changed after capture_graph(): re-capture before reloading weights")
            eng = None
        if eng is None:
            eng = _Engine(self, device, H, W)
            eng.version = self._param_version
            self._engines[key] = eng
        return eng

    def forward(self, x, targets=None, augment=False, cfg=None, _workspace=None):
        """x [B,3,H,W] float (BGR, 0..255), H and W multiples of 32, on CUDA -> {"det_preds": [B, A, 5 + nc]}.
        ``augment=True`` runs the multi-scale test-time augmentation over ``cfg.scales`` (an attribute or a mapping key,
        as the reference's OmegaConf test config carries it) -> {"det_preds": [B, A_tta, 5 + nc]}, the scales' anchors
        in scale order.  Without scales there is nothing to run: the reference defines no default set."""
        scales = tta_scales(cfg) if augment else None
        if augment and scales is None:
            raise NotImplementedError("augment=True needs cfg.scales (the reference's test.scales); there is no default")
        if self.training:
            raise NotImplementedError("YOLOX here is inference only (no training losses)")
        if not torch.is_tensor(x) or not x.is_cuda:
            raise _lib.GdrnError("YOLOX.forward needs a CUDA tensor (no CPU fallback)")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"YOLOX.forward expects [B,3,H,W], got {tuple(x.shape)}")
        B, _, H, W = x.shape
        if H % 32 or W % 32 or H < 32 or W < 32:
            raise ValueError(f"YOLOX input size must be a positive multiple of 32, got {H}x{W}")
        x = x.detach().to(torch.float32).contiguous()
        with torch.cuda.device(x.device):
            eng = self._engine(x.device, H, W)
            tta = scales is not None
            if tta:
                eng.set_scales(scales)
            det = torch.empty((B, eng.A_tta if tta else eng.A, 5 + self.num_classes), dtype=torch.float32, device=x.device)
            ws = _workspace if _workspace is not None else eng.workspace
            if ws is None or ws.numel() < eng.workspace_bytes(B, tta):
                ws = eng.workspace = eng.new_workspace(B, tta)
            eng.run(x, det, ws, tta)   # batches above max_batch run in chunks inside the engine
        return {"det_preds": det}

    def capture_graph(self, x, warmup=2, augment=False, cfg=None):
        """Capture one forward over the static input ``x`` into a CUDA graph -> ``(replay, out_dict)``: ``replay()``
        re-runs the forward as one graph launch on the current stream; refill ``x`` in place between replays.
        ``augment`` / ``cfg`` as in ``forward``: the multi-scale forward replays as one graph too."""
        if not (torch.is_tensor(x) and x.is_cuda and x.is_contiguous() and x.dtype == torch.float32):
            raise _lib.GdrnError("capture_graph: x must be a contiguous float32 CUDA tensor")
        if x.shape[0] > self.max_batch:
            raise _lib.GdrnError(f"capture_graph: batch {x.shape[0]} above max_batch={self.max_batch}")
        with torch.cuda.device(x.device):
            self.forward(x, augment=augment, cfg=cfg)   # builds the engine and its plans outside the capture
            # the graph bakes the workspace pointer in: it gets a workspace of its own, kept alive by replay()
            ws = self._engines[(x.shape[2], x.shape[3])].new_workspace(x.shape[0], tta=bool(augment))
            side = torch.cuda.Stream(device=x.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(warmup):
                    self.forward(x, augment=augment, cfg=cfg, _workspace=ws)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self.forward(x, augment=augment, cfg=cfg, _workspace=ws)
        self._graph_pinned = True

        def replay(_graph=graph, _ws=ws):
            _graph.replay()

        return replay, out


def tta_scales(cfg):
    """The test-time-augmentation scales of a test config (``cfg.scales`` or ``cfg["scales"]``) as a tuple of Python
    floats, or None when there are none."""
    if cfg is None:
        return None
    scales = cfg.get("scales") if isinstance(cfg, Mapping) else getattr(cfg, "scales", None)
    if scales is None:
        return None
    scales = tuple(float(s) for s in scales)
    if not scales:
        raise ValueError("cfg.scales is empty")
    return scales


# ---------------------------------------------------------------------------------------------------------------------
# LazyConfig reader
# ---------------------------------------------------------------------------------------------------------------------
_MODEL_DEFAULTS = {"backbone.depth": 1.0, "backbone.width": 1.0, "backbone.in_channels": [256, 512, 1024],
                   "backbone.depthwise": False, "backbone.act": "silu", "head.num_classes": 80,
                   "head.width": "${..backbone.width}", "head.in_channels": "${..backbone.in_channels}",
                   "head.depthwise": False, "head.act": "silu", "head.strides": [8, 16, 32]}
_TEST_KEYS = ("test_size", "conf_thr", "nms_thr")
_TEST_OPTIONAL = {"augment": False, "scales": None}   # test-time augmentation, off unless the config sets it


def _literal(node, path):
    try:
        return ast.literal_eval(node)
    except ValueError:
        raise ValueError(f"{path}: {ast.unparse(node)!r} is not a literal the config reader can evaluate") from None


def _dotted(node):
    parts = []
    while isinstance(node, ast.Attribute):
        parts.append(node.attr)
        node = node.value
    if isinstance(node, ast.Name):
        parts.append(node.id)
        return ".".join(reversed(parts))
    return None


def _read_config(path, seen):
    path = os.path.abspath(path)
    if path in seen:
        raise ValueError(f"{path}: import cycle")
    seen = seen | {path}
    tree = ast.parse(open(path).read(), path)
    model, test = {}, {}
    for node in tree.body:
        if isinstance(node, ast.ImportFrom) and node.level == 1 and node.module:
            names = {a.name for a in node.names}
            if names & {"model", "test"}:
                base = os.path.join(os.path.dirname(path), *node.module.split(".")) + ".py"
                bm, bt = _read_config(base, seen)
                model.update(bm)
                test.update(bt)
            continue
        if isinstance(node, ast.Assign) and len(node.targets) == 1:
            tgt, val = _dotted(node.targets[0]), node.value
        elif isinstance(node, ast.AnnAssign):
            tgt, val = _dotted(node.target), node.value
        elif isinstance(node, ast.Expr) and isinstance(node.value, ast.Call) and _dotted(node.value.func) in (
                "model.update", "test.update", "model.backbone.update", "model.head.update"):
            obj = _dotted(node.value.func)[:-len(".update")]
            for kw in node.value.keywords:
                _set(model, test, f"{obj}.{kw.arg}", kw.value, path)
            continue
        else:
            continue
        if tgt is None:
            continue
        if tgt == "model":
            model = {}
            _read_lazy_call(val, "", model, path)
        elif tgt == "test":
            if isinstance(val, ast.Call) and _dotted(val.func) == "dict":
                test = {}
                for kw in val.keywords:
                    if kw.arg in _TEST_KEYS or kw.arg in _TEST_OPTIONAL:
                        test[kw.arg] = _literal(kw.value, f"{path}: test.{kw.arg}")
            # test = OmegaConf.create(test) and similar wrappers keep the values
        elif tgt.startswith(("model.", "test.")):
            _set(model, test, tgt, val, path)
    return model, test


def _set(model, test, tgt, val, path):
    if tgt.startswith("model."):
        key = tgt[len("model."):]
        if isinstance(val, ast.Call):
            _read_lazy_call(val, key + ".", model, path)
        else:
            model[key] = _literal(val, f"{path}: {tgt}")
    elif tgt.startswith("test.") and (tgt[len("test."):] in _TEST_KEYS or tgt[len("test."):] in _TEST_OPTIONAL):
        test[tgt[len("test."):]] = _literal(val, f"{path}: {tgt}")


def _read_lazy_call(node, prefix, out, path):
    """model = L(YOLOX)(backbone=L(YOLOPAFPN)(depth=..., ...), head=L(YOLOXHead)(...)): keyword arguments by path."""
    if not isinstance(node, ast.Call):
        raise ValueError(f"{path}: model{('.' + prefix[:-1]) if prefix else ''} is not a LazyCall")
    for kw in node.keywords:
        if isinstance(kw.value, ast.Call) and isinstance(kw.value.func, ast.Call):
            _read_lazy_call(kw.value, prefix + kw.arg + ".", out, path)
        else:
            out[prefix + kw.arg] = _literal(kw.value, f"{path}: model.{prefix}{kw.arg}")


def load_yolox_config(path):
    """Read a reference YOLOX LazyConfig (configs/yolox/**.py) without executing it: the literal assignments to
    model.backbone.depth / width, model.head.num_classes and test.test_size / conf_thr / nms_thr / augment / scales, following the
    ``from .yolox_base import ...`` chain.  A model setting the engine cannot honour (depthwise convs, an activation
    other than silu, other strides or channel lists, a head width other than the backbone's) raises ValueError.
    -> SimpleNamespace(depth, width, num_classes, test_size (h, w), conf_thr, nms_thr, augment (default False),
    scales (a tuple, default None), the test-loop settings and the training loader's (``_train_loader_settings``)).  The
    namespace is also the ``cfg`` of ``YOLOX.forward(augment=True, cfg=cfg)``."""
    model, test = _read_config(path, frozenset())
    cfg = dict(_MODEL_DEFAULTS)
    for k, v in model.items():
        if k not in cfg:
            raise ValueError(f"{path}: model.{k} = {v!r} is not supported by the YOLOX engine")
        cfg[k] = v
    bad = []
    for k in ("backbone.depthwise", "head.depthwise"):
        if cfg[k]:
            bad.append(f"model.{k} = {cfg[k]!r} (depthwise YOLOX is not supported)")
    for k in ("backbone.act", "head.act"):
        if cfg[k] != "silu":
            bad.append(f"model.{k} = {cfg[k]!r} (only silu)")
    if list(cfg["backbone.in_channels"]) != [256, 512, 1024]:
        bad.append(f"model.backbone.in_channels = {cfg['backbone.in_channels']!r}")
    if cfg["head.in_channels"] not in ("${..backbone.in_channels}", [256, 512, 1024]):
        bad.append(f"model.head.in_channels = {cfg['head.in_channels']!r}")
    if cfg["head.width"] not in ("${..backbone.width}", cfg["backbone.width"]):
        bad.append(f"model.head.width = {cfg['head.width']!r} differs from the backbone width")
    if list(cfg["head.strides"]) != [8, 16, 32]:
        bad.append(f"model.head.strides = {cfg['head.strides']!r}")
    if bad:
        raise ValueError(f"{path}: " + "; ".join(bad))
    missing = [k for k in _TEST_KEYS if k not in test]
    if missing:
        raise ValueError(f"{path}: test.{', test.'.join(missing)} not found")
    ex = _read_test_loop_settings(path, frozenset())
    output_dir = ex.get("output_dir")
    if output_dir is None:   # train.output_dir = osp.abspath(__file__).replace("configs", "output", 1)[0:-3]
        output_dir = os.path.abspath(path).replace("configs", "output", 1)[0:-3]
    return SimpleNamespace(depth=float(cfg["backbone.depth"]), width=float(cfg["backbone.width"]),
                           num_classes=int(cfg["head.num_classes"]), test_size=tuple(int(v) for v in test["test_size"]),
                           conf_thr=float(test["conf_thr"]), nms_thr=float(test["nms_thr"]),
                           augment=bool(test.get("augment", _TEST_OPTIONAL["augment"])),
                           scales=None if test.get("scales") is None else tuple(test["scales"]),
                           test_dataset_names=tuple(ex.get("test_dataset_names", ())),
                           half_test=bool(ex.get("half_test", False)), amp_test=bool(ex.get("amp_test", False)),
                           output_dir=output_dir, eval_cached=bool(ex.get("eval_cached", False)),
                           legacy=bool(ex.get("legacy", False)), filter_scene=bool(ex.get("filter_scene", False)),
                           **_train_loader_settings(path))


# MosaicDetection's keyword defaults (det/yolox/data/datasets/mosaicdetection.py)
_AUG_WRAPPER_DEFAULTS = {"mosaic": True, "degrees": 10.0, "translate": 0.1, "mosaic_scale": (0.5, 1.5),
                         "mixup_scale": (0.5, 1.5), "shear": 2.0, "enable_mixup": True, "mosaic_prob": 1.0,
                         "mixup_prob": 1.0, "COLOR_AUG_PROB": 0.0, "COLOR_AUG_TYPE": "", "COLOR_AUG_CODE": (),
                         "AUG_HSV_PROB": 0, "HSV_H": 0, "HSV_S": 0, "HSV_V": 0, "FORMAT": "RGB",
                         "preproc.max_labels": 50, "preproc.flip_prob": 0.5, "preproc.hsv_prob": 1.0}


def _train_loader_settings(path):
    """The training loader of the config (dataloader.train = L(build_yolox_train_loader)(...) and the
    dataloader.train.* assignments after it), DATASETS.TRAIN and train.no_aug_epochs -> train_img_size (h, w),
    train_dataset_names, aug_wrapper (MosaicDetection's keywords with their defaults, preproc.* for its TrainTransform),
    train_total_batch_size, train_num_workers, no_aug_epochs."""
    flat = _read_train_settings(path, frozenset())
    wrap = dict(_AUG_WRAPPER_DEFAULTS)
    wrap.update({k[len("aug_wrapper."):]: v for k, v in flat.items() if k.startswith("aug_wrapper.")})
    size = flat.get("dataset.img_size", (416, 416))   # Base_DatasetFromList's default
    if wrap.get("img_size", "${..dataset.img_size}") != "${..dataset.img_size}":
        size = wrap["img_size"]
    wrap.pop("img_size", None)
    return {"train_img_size": tuple(int(v) for v in size), "train_dataset_names": tuple(flat.get("DATASETS.TRAIN", ())),
            "aug_wrapper": wrap, "train_total_batch_size": int(flat.get("total_batch_size", 64)),
            "train_num_workers": int(flat.get("num_workers", 0)), "no_aug_epochs": int(flat.get("train.no_aug_epochs", 0))}


def _read_train_settings(path, seen):
    path = os.path.abspath(path)
    if path in seen:
        raise ValueError(f"{path}: import cycle")
    tree = ast.parse(open(path).read(), path)
    out = {}

    def lit(node):
        try:
            return ast.literal_eval(node)
        except ValueError:
            return None

    def call_kwargs(node, prefix):
        for kw in node.keywords:
            if isinstance(kw.value, ast.Call) and isinstance(kw.value.func, ast.Call):
                call_kwargs(kw.value, f"{prefix}{kw.arg}.")
            else:
                v = lit(kw.value)
                if v is not None:
                    out[prefix + kw.arg] = v

    for node in tree.body:
        if isinstance(node, ast.ImportFrom) and node.level == 1 and node.module:
            base = os.path.join(os.path.dirname(path), *node.module.split(".")) + ".py"
            if os.path.exists(base) and {a.name for a in node.names} & {"dataloader", "train", "DATASETS"}:
                out.update(_read_train_settings(base, seen | {path}))
            continue
        if isinstance(node, ast.Expr) and isinstance(node.value, ast.Call) and _dotted(node.value.func) == "train.update":
            for kw in node.value.keywords:
                if kw.arg == "no_aug_epochs" and lit(kw.value) is not None:
                    out["train.no_aug_epochs"] = lit(kw.value)
            continue
        if not (isinstance(node, ast.Assign) and len(node.targets) == 1):
            continue
        tgt, val = _dotted(node.targets[0]), node.value
        if tgt == "dataloader.train" and isinstance(val, ast.Call):
            out = {k: v for k, v in out.items() if not k.startswith(("dataset.", "aug_wrapper.", "total_batch_size",
                                                                     "num_workers"))}
            call_kwargs(val, "")
        elif tgt and tgt.startswith("dataloader.train."):
            v = lit(val)
            if v is not None:
                out[tgt[len("dataloader.train."):]] = v
        elif tgt in ("train", "DATASETS") and isinstance(val, ast.Call) and _dotted(val.func) == "dict":
            for kw in val.keywords:
                if (tgt, kw.arg) in (("train", "no_aug_epochs"), ("DATASETS", "TRAIN")) and lit(kw.value) is not None:
                    out[f"{tgt}.{kw.arg}"] = lit(kw.value)
        elif tgt in ("train.no_aug_epochs", "DATASETS.TRAIN") and lit(val) is not None:
            out[tgt] = lit(val)
    return out


def _read_test_loop_settings(path, seen):
    """The settings of the dataset test loop (main_yolox.py --eval-only) along the import chain: DATASETS.TEST /
    test.test_dataset_names, test.half_test / amp_test, val.eval_cached, a literal train.output_dir, and the
    ValTransform(legacy=...) / YOLOX_COCOEvaluator(filter_scene=...) arguments of the test loaders."""
    path = os.path.abspath(path)
    if path in seen:
        raise ValueError(f"{path}: import cycle")
    tree = ast.parse(open(path).read(), path)
    out = {}

    def lit(node, default=None):
        try:
            return ast.literal_eval(node)
        except ValueError:
            return default

    for node in tree.body:
        if isinstance(node, ast.ImportFrom) and node.level == 1 and node.module:
            base = os.path.join(os.path.dirname(path), *node.module.split(".")) + ".py"
            if os.path.exists(base) and {a.name for a in node.names} & {"test", "DATASETS", "train", "val"}:
                out.update(_read_test_loop_settings(base, seen | {path}))
            continue
        if isinstance(node, ast.Assign) and len(node.targets) == 1:
            tgt, val = _dotted(node.targets[0]), node.value
            if tgt in ("test", "val", "train", "DATASETS") and isinstance(val, ast.Call) and _dotted(val.func) == "dict":
                for kw in val.keywords:
                    _test_loop_key(out, f"{tgt}.{kw.arg}", kw.value, lit)
            elif tgt:
                _test_loop_key(out, tgt, val, lit)
        elif isinstance(node, ast.Expr) and isinstance(node.value, ast.Call) and _dotted(node.value.func) in (
                "train.update", "test.update", "val.update"):
            obj = _dotted(node.value.func)[:-len(".update")]
            for kw in node.value.keywords:
                _test_loop_key(out, f"{obj}.{kw.arg}", kw.value, lit)
        for sub in ast.walk(node):
            if isinstance(sub, ast.Call) and isinstance(sub.func, ast.Call) and sub.func.args:
                name = _dotted(sub.func.args[0])   # L(ValTransform)(legacy=...)
                for kw in sub.keywords:
                    if name == "ValTransform" and kw.arg == "legacy":
                        out["legacy"] = bool(lit(kw.value, True))
                    elif name == "YOLOX_COCOEvaluator" and kw.arg == "filter_scene":
                        out["filter_scene"] = bool(lit(kw.value, True))
    return out


def _test_loop_key(out, tgt, val, lit):
    if tgt == "DATASETS.TEST":
        names = lit(val)
        if names is not None:
            out["datasets_test"] = tuple(names)
            out["test_dataset_names"] = tuple(names)
    elif tgt == "test.test_dataset_names":
        names = out.get("datasets_test", ()) if _dotted(val) == "DATASETS.TEST" else lit(val)
        if names is not None:
            out["test_dataset_names"] = tuple(names)
    elif tgt in ("test.half_test", "test.amp_test", "val.eval_cached"):
        out[tgt.split(".")[1]] = bool(lit(val, True))
    elif tgt == "train.output_dir":
        v = lit(val)
        out["output_dir"] = v if isinstance(v, str) else None
