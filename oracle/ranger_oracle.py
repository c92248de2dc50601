"""Oracle of the Ranger step and the model-EMA update (gdrnpp_bop2022_b200/ranger.py, ema.py).

``RefRanger`` restates the reference's ``Ranger.step`` (lib/torch_utils/solver/ranger.py) as the same sequence of
torch ops, in the dtype of the parameters (fp32 reproduces the reference; fp64 is the accuracy yardstick), with the
reference's constructor, attributes and state keys, so that state dicts move between it and the fused class.
``ema_update`` restates ``ModelEMA.update``'s two ops per entry.

Seeded case builders: ``CASES`` names the parameter sets, groups and hyper-parameters; ``make_params`` draws the
initial parameters, ``grad_at`` the gradient of a parameter at a step (None on the steps listed in ``no_grad``),
``lr_at`` the learning rate of a group at a step; ``run_case`` drives any Ranger-shaped class through them.
``sample_positions`` gives the seeded flat positions stored in tests/golden/ref_ranger.npz.
"""
import math

import numpy as np
import torch
from torch.optim.optimizer import Optimizer

N_SAMPLES = 48
GOLDEN_STEPS = (5, 6, 7, 12, 14)
STATE_KEYS = ("exp_avg", "exp_avg_sq", "slow_buffer")
RESUME_CASE, RESUME_STEP, LAST_STEP = "options", 7, 14
EMA_CASES = ((0.9998, 0), (0.9998, 3000))   # (decay, initial updates) of the stored EMAs

# name -> dict(opt = constructor kwargs, groups = [(group kwargs, [(param name, shape), ...]), ...],
#              no_grad = {param name: steps without a gradient})
CASES = {
    "gdrn": dict(
        opt=dict(lr=8e-4, weight_decay=0.01),
        groups=[
            (dict(lr=8e-4), [("stem.weight", (32, 3, 4, 4)), ("stem.bias", (32,)), ("dw.weight", (32, 1, 7, 7)),
                             ("dw.bias", (32,)), ("norm.weight", (32,)), ("norm.bias", (32,)),
                             ("fc1.weight", (128, 32)), ("fc1.bias", (128,)), ("fc2.weight", (32, 128)),
                             ("gamma", (32,)), ("deconv.weight", (32, 16, 3, 3))]),
            (dict(lr=4e-4), [("head.weight", (24, 16, 3, 3)), ("gn.weight", (24,)), ("pnp_fc1.weight", (6, 8192)),
                             ("pnp_fc1.bias", (6,)), ("fc_r.weight", (6, 256))]),
        ],
        no_grad={"gamma": (3, 9)},
    ),
    "yolox": dict(
        opt=dict(lr=0.001, weight_decay=0),
        groups=[
            (dict(), [("bn0.weight", (48,)), ("bn0.bias", (48,)), ("bn1.weight", (96,)), ("bn1.bias", (96,))]),
            (dict(), [("stem.conv.weight", (48, 12, 3, 3)), ("dark2.conv.weight", (96, 48, 3, 3)),
                      ("cv1.conv.weight", (48, 96, 1, 1)), ("cls_preds.weight", (8, 96, 1, 1))]),
            (dict(), [("cls_preds.bias", (8,)), ("reg_preds.bias", (4,))]),
        ],
        no_grad={},
    ),
    "options": dict(
        opt=dict(lr=1e-3, alpha=0.8, k=4, N_sma_threshhold=4, weight_decay=0.01, use_gc=False, gc_conv_only=True),
        groups=[
            (dict(), [("conv.weight", (16, 8, 3, 3)), ("fc.weight", (24, 40)), ("fc.bias", (24,))]),
            (dict(betas=(0.9, 0.99), lr=2e-3), [("conv2.weight", (8, 16, 3, 3)), ("fc2.weight", (10, 24)),
                                                 ("bn.weight", (8,))]),
        ],
        no_grad={},
    ),
}


def _seed(*parts):
    return int(np.random.default_rng([len(parts), *[sum(map(ord, str(p))) * 131 + i for i, p in enumerate(parts)]])
               .integers(0, 2**62))


def param_names(case):
    return [name for _, params in CASES[case]["groups"] for name, _ in params]


def param_shapes(case):
    return {name: shape for _, params in CASES[case]["groups"] for name, shape in params}


def initial_param(case, name, shape):
    """fp32 CPU values: weights ~ N(0, 0.05), 1-D norms around 1, biases ~ N(0, 0.02)."""
    g = torch.Generator().manual_seed(_seed(case, name, "init"))
    x = torch.randn(shape, generator=g, dtype=torch.float32)
    if len(shape) == 1:
        return (1.0 + 0.1 * x) if ("norm" in name or "bn" in name or "gn" in name) else 0.02 * x
    return 0.05 * x


def grad_at(case, name, shape, step):
    """fp32 CPU gradient at ``step`` (1-based), or None.  Each dim-0 slice carries an offset, so GC matters."""
    if step in CASES[case]["no_grad"].get(name, ()):
        return None
    g = torch.Generator().manual_seed(_seed(case, name, "grad", step))
    x = 1e-2 * torch.randn(shape, generator=g, dtype=torch.float32)
    if len(shape) > 1:
        x += 5e-3 * torch.randn((shape[0],) + (1,) * (len(shape) - 1), generator=g, dtype=torch.float32)
    return x


def lr_at(case, group_index, step):
    """Learning rate of a group at ``step``: the group's base lr on a decaying, step-to-step changing schedule."""
    c = CASES[case]
    base = c["groups"][group_index][0].get("lr", c["opt"]["lr"])
    return base * (1.0 - 0.03 * step) * (1.0 + 0.1 * math.sin(step))


def make_params(case, dtype=torch.float32, device="cpu"):
    """[[Parameter, ...] per group] with the seeded initial values, and the optimizer's param_groups argument."""
    groups, arg = [], []
    for gkw, params in CASES[case]["groups"]:
        ps = [torch.nn.Parameter(initial_param(case, n, s).to(device=device, dtype=dtype)) for n, s in params]
        groups.append(ps)
        arg.append(dict(gkw, params=ps))
    return groups, arg


def set_grads(case, groups, step, dtype=None):
    for (_, params), ps in zip(CASES[case]["groups"], groups):
        for (name, shape), p in zip(params, ps):
            g = grad_at(case, name, shape, step)
            p.grad = None if g is None else g.to(device=p.device, dtype=dtype or p.dtype)


def set_lrs(case, opt, step):
    for gi, group in enumerate(opt.param_groups):
        group["lr"] = lr_at(case, gi, step)


def run_case(case, opt_cls, dtype=torch.float32, device="cpu", steps=LAST_STEP, on_step=None):
    """Run steps 1..steps; ``on_step(step, groups, opt)`` after each.  Returns (groups, opt)."""
    groups, arg = make_params(case, dtype, device)
    opt = opt_cls(arg, **CASES[case]["opt"])
    for step in range(1, steps + 1):
        set_lrs(case, opt, step)
        set_grads(case, groups, step)
        opt.step()
        if on_step is not None:
            on_step(step, groups, opt)
    return groups, opt


def sample_positions(name, shape):
    """The seeded flat positions of a tensor stored in the golden file."""
    rng = np.random.default_rng([len(name), *map(ord, name)])
    return rng.integers(0, int(np.prod(shape)), N_SAMPLES)


def snapshot(case, groups, opt):
    """{(param name, key): tensor} for key in p, exp_avg, exp_avg_sq, slow_buffer, and {param name: step}."""
    vals, steps = {}, {}
    for (_, params), ps in zip(CASES[case]["groups"], groups):
        for (name, _), p in zip(params, ps):
            vals[(name, "p")] = p.detach()
            st = opt.state[p]
            steps[name] = st.get("step", 0)
            for k in STATE_KEYS:
                vals[(name, k)] = st[k] if k in st else torch.zeros_like(p)
    return vals, steps


# ------------------------------------------------------------------------------------- the reference's step
class RefRanger(Optimizer):
    """The reference's Ranger as torch ops in the parameters' dtype (state keys and attributes as the reference)."""

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
        super().__init__(params, dict(lr=lr, alpha=alpha, k=k, step_counter=0, betas=betas,
                                      N_sma_threshhold=N_sma_threshhold, eps=eps, weight_decay=weight_decay))
        self.N_sma_threshhold = N_sma_threshhold
        self.alpha = alpha
        self.k = k
        self.radam_buffer = [[None, None, None] for _ in range(10)]
        self.use_gc = use_gc
        self.gc_gradient_threshold = 3 if gc_conv_only else 1

    def _coefficients(self, step, beta1, beta2):
        slot = self.radam_buffer[step % 10]
        if slot[0] != step:
            b2t = beta2 ** step
            n_max = 2 / (1 - beta2) - 1
            n_sma = n_max - 2 * step * b2t / (1 - b2t)
            if n_sma > self.N_sma_threshhold:
                size = math.sqrt((1 - b2t) * (n_sma - 4) / (n_max - 4) * (n_sma - 2) / n_sma * n_max
                                 / (n_max - 2)) / (1 - beta1 ** step)
            else:
                size = 1.0 / (1 - beta1 ** step)
            slot[:] = [step, n_sma, size]
        return slot[1], slot[2]

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                if g.is_sparse:
                    raise RuntimeError("Ranger optimizer does not support sparse gradients")
                st = self.state[p]
                if not st:
                    st.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p),
                              slow_buffer=p.detach().clone())
                m, v = st["exp_avg"], st["exp_avg_sq"]
                if g.dim() > self.gc_gradient_threshold:   # GC, in place in p.grad
                    g.add_(-(g.mean(dim=tuple(range(1, g.dim())), keepdim=True)))
                st["step"] += 1
                v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
                m.mul_(beta1).add_(g, alpha=1 - beta1)
                n_sma, size = self._coefficients(st["step"], beta1, beta2)
                if group["weight_decay"] != 0:
                    p.add_(p, alpha=-group["weight_decay"] * group["lr"])
                if n_sma > self.N_sma_threshhold:
                    p.addcdiv_(m, v.sqrt().add_(group["eps"]), value=-size * group["lr"])
                else:
                    p.add_(m, alpha=-size * group["lr"])
                if st["step"] % group["k"] == 0:
                    slow = st["slow_buffer"]
                    slow.add_(p - slow, alpha=self.alpha)
                    p.copy_(slow)
        return None


# ------------------------------------------------------------------------------------------------- the EMA
def ema_decay(decay, updates):
    return decay * (1 - math.exp(-updates / 2000))


@torch.no_grad()
def ema_update(ema_sd, model_sd, d):
    """ModelEMA.update's two ops on every floating entry, in place in ``ema_sd``."""
    for k, v in ema_sd.items():
        if v.dtype.is_floating_point:
            v *= d
            v += (1.0 - d) * model_sd[k].detach()


def make_ema_model(seed=0):
    """A small YOLOX-like module: convs with BatchNorm (running stats and num_batches_tracked) and a biased conv."""
    torch.manual_seed(seed)
    nn = torch.nn
    m = nn.Sequential(nn.Conv2d(3, 16, 3, bias=False), nn.BatchNorm2d(16), nn.SiLU(), nn.Conv2d(16, 32, 1, bias=False),
                      nn.BatchNorm2d(32), nn.SiLU(), nn.Conv2d(32, 8, 1))
    return perturb_model(m, seed, 0)


@torch.no_grad()
def perturb_model(model, seed, update):
    """Seeded stand-in for a training step: every floating entry moves, num_batches_tracked counts up."""
    g = torch.Generator().manual_seed(_seed("ema", seed, update))
    for k, v in model.state_dict().items():
        if v.dtype.is_floating_point:
            delta = 0.05 * torch.randn(v.shape, generator=g, dtype=torch.float32).to(v.device)
            v.add_(delta.abs() if k.endswith("running_var") else delta)
        else:
            v += 1
    return model
