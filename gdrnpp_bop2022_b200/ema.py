"""Model EMA as one GPU launch per update: a drop-in for the reference's ``ModelEMA`` (``det/yolox/utils/ema.py``, and
the same formula in ``lib/torch_utils/torch_utils.py``), which the detector trainer updates after every step.

``update`` walks every floating entry of the EMA's state dict (parameters and buffers) in one kernel
(``csrc/train_step.cu``).  Each element is ``fl(fl(v * d32) + fl(c32 * m))`` with ``d32 = fp32(d)`` and
``c32 = fp32(1.0 - d)``, ``d`` computed in double: bit for bit the reference's ``v *= d; v += (1.0 - d) * m``.
Integer entries (``num_batches_tracked``) are left alone.  DESIGN.md §7s.

Bindings: ``det.yolox.engine.yolox_trainer.ModelEMA = ModelEMA`` and ``core.gdrn_modeling.engine.engine.ModelEMA =
ModelEMA`` (INTEGRATION.md §7q).
"""
import ctypes
import math
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .ranger import _dense_dim0_outer

__all__ = ["ModelEMA", "is_parallel", "copy_attr"]


def is_parallel(model):
    return isinstance(model, (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel))


def copy_attr(a, b, include=(), exclude=()):
    """Copy the public attributes of ``b`` onto ``a``, only ``include`` when it is given, never ``exclude``."""
    for k, v in b.__dict__.items():
        if (len(include) and k not in include) or k.startswith("_") or k in exclude:
            continue
        setattr(a, k, v)


class ModelEMA:
    def __init__(self, model, decay=0.9999, updates=0):
        self.ema = deepcopy(model.module if is_parallel(model) else model).eval()
        self.updates = updates
        self.decay = lambda x: decay * (1 - math.exp(-x / 2000))   # ramp for the early updates
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def _pairs(self, model):
        """(ema entry, model entry) for every non-empty floating entry, checked before anything changes."""
        msd = model.module.state_dict() if is_parallel(model) else model.state_dict()
        pairs, device = [], None
        for k, v in self.ema.state_dict().items():
            if not v.dtype.is_floating_point:
                continue
            m = msd[k].detach()
            if v.dtype != torch.float32 or m.dtype != torch.float32:
                raise TypeError(f"ModelEMA: entry {k!r} has dtype {v.dtype} (model: {m.dtype}); the fused update takes "
                                "float32 only")
            if not (v.is_cuda and m.is_cuda):
                raise ValueError(f"ModelEMA: entry {k!r} is not a CUDA tensor in the EMA or in the model")
            device = v.device if device is None else device
            if v.device != device or m.device != device:
                raise ValueError(f"ModelEMA: entry {k!r} is on {v.device} (model: {m.device}), another entry on "
                                 f"{device}; the fused update takes one device")
            if v.shape != m.shape or v.stride() != m.stride() or not _dense_dim0_outer(v):
                raise ValueError(f"ModelEMA: entry {k!r} has shape {tuple(v.shape)} and strides {v.stride()} in the "
                                 f"EMA, {tuple(m.shape)} and {m.stride()} in the model; both must be the same dense "
                                 "layout")
            if v.numel():
                pairs.append((v, m))
        return pairs, device

    def update(self, model):
        with torch.no_grad():
            pairs, device = self._pairs(model)
            self.updates += 1
            d = self.decay(self.updates)
            if not pairs:
                return
            n = len(pairs)
            table = np.zeros((n, 4), np.int64)   # GdrnEmaEntry (include/gdrn_b200.h)
            table[:, :3] = [(v.data_ptr(), m.data_ptr(), v.numel()) for v, m in pairs]
            L = _lib.lib()
            n_units = ctypes.c_longlong()
            _lib.check(L.gdrn_ema_plan(table.ctypes.data, n, ctypes.byref(n_units)), "gdrn_ema_plan")
            with torch.cuda.device(device):
                dev_table = torch.from_numpy(table.reshape(-1)).pin_memory().to(device, non_blocking=True)
                # ctypes rounds each double to fp32 once, as torch does with a Python scalar
                _lib.check(L.gdrn_ema_update(_lib.ptr(dev_table), n, n_units.value, d, 1.0 - d,
                                             _lib.current_stream()), "gdrn_ema_update")

    def update_attr(self, model, include=(), exclude=("process_group", "reducer")):
        copy_attr(self.ema, model, include, exclude)
