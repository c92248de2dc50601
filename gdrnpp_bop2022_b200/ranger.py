"""Ranger (gradient centralisation + RAdam + lookahead) as one fused GPU pass per step: a drop-in for the reference's
``lib/torch_utils/solver/ranger.py:Ranger``, which every shipped GDRN config and the Ranger YOLOX configs train with.

The constructor, ``defaults``, the attributes and the per-parameter state (``step`` as a Python int, ``exp_avg``,
``exp_avg_sq``, ``slow_buffer``) are the reference's, so checkpoints move between the two classes in both directions.
``step()`` keeps the host work the reference does per tensor (step counters, the shared ``radam_buffer`` cache, the
fp32 scalars), writes one descriptor per parameter, uploads the table and issues one update kernel
(``csrc/train_step.cu``; a second, the long-row means pass, only when a parameter has dim-0 slices longer than 8192
elements).  The number of launches does not depend on the number of tensors.  DESIGN.md §7s pins every rule.

Bindings into the reference: ``OPTIMIZERS.register_module()(Ranger)`` for GDRN, ``lib.torch_utils.solver.ranger.Ranger
= Ranger`` before the YOLOX LazyConfig is loaded (INTEGRATION.md §7q).
"""
import ctypes
import math

import numpy as np
import torch
from torch.optim.optimizer import Optimizer

from . import _lib

# GdrnRangerParam (include/gdrn_b200.h): 16 eight-byte words per parameter
_WORDS = 16
_F_GC, _F_INIT, _F_WD, _F_ADAPTIVE, _F_LOOKAHEAD = 1, 2, 4, 8, 16


def _dense_dim0_outer(t):
    """True when ``t`` covers one dense block and each dim-0 slice is one dense block (contiguous, channels_last)."""
    if t.is_contiguous() or (t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)) or t.numel() <= 1:
        return True
    dims = sorted((st, sz) for sz, st in zip(t.shape, t.stride()) if sz != 1)
    expected = 1
    for st, sz in dims:
        if st != expected:
            return False
        expected *= sz
    return t.shape[0] == 1 or t.stride(0) == t.numel() // t.shape[0]


def _where(gi, pi, p):
    return f"parameter {pi} of param group {gi} (shape {tuple(p.shape)})"


class Ranger(Optimizer):
    def __init__(self, params, lr=1e-3, alpha=0.5, k=6, N_sma_threshhold=5, betas=(0.95, 0.999), eps=1e-5,
                 weight_decay=0, use_gc=True, gc_conv_only=False):
        if not 0.0 <= alpha <= 1.0:
            raise ValueError(f"Invalid slow update rate: {alpha}")
        if not 1 <= k:
            raise ValueError(f"Invalid lookahead steps: {k}")
        if not lr > 0:
            raise ValueError(f"Invalid Learning Rate: {lr}")
        if not eps > 0:
            raise ValueError(f"Invalid eps: {eps}")
        defaults = dict(lr=lr, alpha=alpha, k=k, step_counter=0, betas=betas, N_sma_threshhold=N_sma_threshhold,
                        eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.N_sma_threshhold = N_sma_threshhold
        self.alpha = alpha
        self.k = k
        # (step, N_sma, step_size) per step % 10, shared by every group, as in the reference
        self.radam_buffer = [[None, None, None] for _ in range(10)]
        # Stored as the reference stores it.  The reference's step never reads it: GC follows the dimension rule alone.
        self.use_gc = use_gc
        self.gc_gradient_threshold = 3 if gc_conv_only else 1

    def _radam(self, step, beta1, beta2):
        """N_sma and step_size of this step through the shared radam_buffer, in the reference's order."""
        buffered = self.radam_buffer[int(step % 10)]
        if step == buffered[0]:
            return buffered[1], buffered[2]
        beta2_t = beta2 ** step
        n_max = 2 / (1 - beta2) - 1
        n_sma = n_max - 2 * step * beta2_t / (1 - beta2_t)
        if n_sma > self.N_sma_threshhold:
            ratio = (1 - beta2_t) * (n_sma - 4) / (n_max - 4) * (n_sma - 2) / n_sma * n_max / (n_max - 2)
            step_size = math.sqrt(ratio) / (1 - beta1 ** step)
        else:
            step_size = 1.0 / (1 - beta1 ** step)
        buffered[:] = [step, n_sma, step_size]
        return n_sma, step_size

    def _collect(self):
        """Every (group index, index in group, group, parameter) with a gradient, checked before any state changes."""
        items, device = [], None
        for gi, group in enumerate(self.param_groups):
            for pi, p in enumerate(group["params"]):
                g = p.grad
                if g is None:
                    continue
                if g.is_sparse:
                    raise RuntimeError("Ranger optimizer does not support sparse gradients")
                if p.dtype != torch.float32 or g.dtype != torch.float32:
                    raise TypeError(f"Ranger: {_where(gi, pi, p)} has dtype {p.dtype} and gradient dtype {g.dtype}; "
                                    "the fused step takes float32 only")
                if g.stride() != p.stride():
                    raise ValueError(f"Ranger: {_where(gi, pi, p)} has strides {p.stride()} but its gradient has "
                                     f"{g.stride()}")
                if not _dense_dim0_outer(p):
                    raise ValueError(f"Ranger: {_where(gi, pi, p)} with strides {p.stride()} is not one dense block "
                                     "with dim 0 outermost")
                if not (p.is_cuda and g.is_cuda):
                    raise ValueError(f"Ranger: {_where(gi, pi, p)} or its gradient is not a CUDA tensor")
                if device is None:
                    device = p.device
                if p.device != device or g.device != device:
                    raise ValueError(f"Ranger: {_where(gi, pi, p)} is on {p.device} (gradient on {g.device}), another "
                                     f"parameter on {device}; the fused step takes one device")
                items.append((gi, pi, group, p))
        return items, device

    @staticmethod
    def _state_ptr(state, key, p, stride):
        """Address of a state tensor in the parameter's dtype, device and strides (a loaded checkpoint may differ)."""
        t = state[key]
        if t.dtype is not torch.float32 or t.stride() != stride or t.get_device() != p.get_device():
            t = state[key] = torch.empty_like(p).copy_(t)
        return t.data_ptr()

    @torch.no_grad()
    def step(self, closure=None):
        items, device = self._collect()
        if not items:
            return None
        n = len(items)
        words, scalars, flag_list = [], [], []
        for gi, pi, group, p in items:
            state = self.state[p]
            flags = 0
            if len(state) == 0:
                state["step"] = 0
                state["exp_avg"] = torch.empty_like(p)      # zeroed by the kernel (flag 2)
                state["exp_avg_sq"] = torch.empty_like(p)
                state["slow_buffer"] = torch.empty_like(p)  # the parameter before this step, written by the kernel
                flags |= _F_INIT
            stride = p.stride()
            ptrs = (p.data_ptr(), p.grad.data_ptr(), self._state_ptr(state, "exp_avg", p, stride),
                    self._state_ptr(state, "exp_avg_sq", p, stride), self._state_ptr(state, "slow_buffer", p, stride))
            beta1, beta2 = group["betas"]
            if p.dim() > self.gc_gradient_threshold:
                flags |= _F_GC
            state["step"] += 1
            n_sma, step_size = self._radam(state["step"], beta1, beta2)
            if group["weight_decay"] != 0:
                flags |= _F_WD
            if n_sma > self.N_sma_threshhold:
                flags |= _F_ADAPTIVE
            if state["step"] % group["k"] == 0:
                flags |= _F_LOOKAHEAD
            numel = p.numel()
            words.append(ptrs + (numel, numel // p.shape[0] if p.dim() and p.shape[0] else numel))
            flag_list.append(flags)
            # each scalar rounded once from the double the reference passes to torch
            scalars.append((beta1, 1 - beta1, beta2, 1 - beta2, -step_size * group["lr"],
                            -group["weight_decay"] * group["lr"], group["eps"], self.alpha))
        table = np.zeros((n, _WORDS), np.int64)
        table[:, :7] = words
        table.view(np.int32)[:, 19] = flag_list
        table.view(np.float32)[:, 20:28] = scalars
        L = _lib.lib()
        n_units, n_long = ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.gdrn_ranger_plan(table.ctypes.data, n, ctypes.byref(n_units), ctypes.byref(n_long)),
                   "gdrn_ranger_plan")
        if n_units.value == 0:
            return None
        with torch.cuda.device(device):
            # pinned staging from torch's caching host allocator: it is not reused before the copy has run
            dev_table = torch.from_numpy(table.reshape(-1)).pin_memory().to(device, non_blocking=True)
            ws_bytes = L.gdrn_ranger_workspace_bytes(n_long.value)
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
            _lib.check(L.gdrn_ranger_step(_lib.ptr(dev_table), n, n_units.value, n_long.value, _lib.ptr(ws), ws_bytes,
                                          _lib.current_stream()), "gdrn_ranger_step")
        return None
