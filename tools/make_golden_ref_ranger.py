"""Generate tests/golden/ref_ranger.npz by running the REFERENCE's own ``Ranger`` (lib/torch_utils/solver/ranger.py)
and ``ModelEMA`` (det/yolox/utils/ema.py), imported read-only from the checkout that GDRN_REFERENCE_SRC names with the
import stubs of make_golden_ref_heads.py, on the CPU in fp32.

Inputs are not stored: ``oracle.ranger_oracle`` regenerates the parameters, gradients, learning rates and missing
gradients of each case from its seeds.  Stored (keys ``<case>/<step>/...``) at the steps of GOLDEN_STEPS: per
parameter and per state (p, exp_avg, exp_avg_sq, slow_buffer) the fp64 sum and the values at the seeded positions of
``oracle.ranger_oracle.sample_positions``, and every parameter's step counter.  The full state of the RESUME_CASE at
RESUME_STEP (parameters and the reference's state_dict tensors) under ``resume/``, and two EMAs of a small YOLOX-like
module after three updates in full under ``ema<i>/``.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_ref_ranger.py
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
sys.path.insert(0, ROOT)

from oracle import ranger_oracle as O  # noqa: E402


def load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def record(case, data):
    def on_step(step, groups, opt):
        if step not in O.GOLDEN_STEPS:
            return
        vals, steps = O.snapshot(case, groups, opt)
        for (name, key), t in vals.items():
            t = t.numpy()
            data[f"{case}/{step}/{name}/{key}/sum"] = np.float64(t.astype(np.float64).sum())
            data[f"{case}/{step}/{name}/{key}/samp"] = t.reshape(-1)[O.sample_positions(f"{case}/{name}/{key}",
                                                                                    t.shape)]
        data[f"{case}/{step}/steps"] = np.array([steps[n] for n in O.param_names(case)], np.int64)
        if case == O.RESUME_CASE and step == O.RESUME_STEP:
            sd = opt.state_dict()
            flat = [p for ps in groups for p in ps]
            for i, p in enumerate(flat):
                data[f"resume/p/{i}"] = p.detach().numpy().copy()
                st = sd["state"][i]
                data[f"resume/step/{i}"] = np.int64(st["step"])
                for k in O.STATE_KEYS:
                    data[f"resume/{k}/{i}"] = st[k].numpy().copy()

    return on_step


def main():
    assert REF and os.path.isdir(REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_ref_heads as mh

    sys.meta_path.insert(0, mh.StubFinder())
    sys.path.insert(0, REF)
    Ranger = load("ref_ranger", "lib/torch_utils/solver/ranger.py").Ranger
    ModelEMA = load("ref_ema", "det/yolox/utils/ema.py").ModelEMA
    torch.set_num_threads(1)

    data = {}
    for case in O.CASES:
        groups, opt = O.run_case(case, Ranger, on_step=record(case, data))
        keys = set(k for st in opt.state_dict()["state"].values() for k in st)
        assert keys == {"step", *O.STATE_KEYS}, keys
        print(case, "steps", data[f"{case}/{O.LAST_STEP}/steps"])
    for i, (decay, updates) in enumerate(O.EMA_CASES):
        model = O.make_ema_model(seed=i)
        ema = ModelEMA(model, decay, updates)
        for u in range(3):
            O.perturb_model(model, i, u + 1)
            ema.update(model)
        data[f"ema{i}/updates"] = np.int64(ema.updates)
        for k, v in ema.ema.state_dict().items():
            data[f"ema{i}/{k}"] = v.numpy().copy()
    path = os.path.join(ROOT, "tests", "golden", "ref_ranger.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
