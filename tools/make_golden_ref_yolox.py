"""Generate tests/golden/ref_yolox.npz by running the REFERENCE's own YOLOX (det/yolox/models: YOLOX(YOLOPAFPN, YOLOXHead),
imported read-only from the checkout that GDRN_REFERENCE_SRC names, with the import stubs of make_golden_ref_heads.py)
on a small seeded input.

Small model: depth 0.33, width 0.25, 3 classes, input 2 x 3 x 64 x 96 (0..255).  Weights and BatchNorm statistics are
not stored: they are drawn from a seeded generator in state-dict order by ``draw_state_dict`` (tests/test_yolox.py
repeats it from the stored names and shapes).  Only the input, det_preds and the names / shapes are stored.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_ref_yolox.py
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
DEPTH, WIDTH, NC = 0.33, 0.25, 3


def draw_state_dict(names, shapes, seed=1):
    """Seeded weights in state-dict order: conv weights N(0, 1/fan_in) (the stem's scaled by 1/255 for the 0..255
    input), BatchNorm weight U(0.8, 1.2), bias / running_mean N(0, 0.1), running_var U(0.75, 1.25), conv biases
    N(0, 0.1); num_batches_tracked = 0."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for n, s in zip(names, shapes):
        shape = tuple(int(d) for d in s.split(",")) if s else ()
        if n.endswith("num_batches_tracked"):
            sd[n] = torch.zeros((), dtype=torch.int64)
        elif len(shape) == 4:
            std = math.sqrt(1.0 / (shape[1] * shape[2] * shape[3]))
            if n.endswith("stem.conv.conv.weight"):
                std /= 255.0
            sd[n] = torch.randn(shape, generator=g, dtype=torch.float64).float() * std
        elif n.endswith("bn.weight"):
            sd[n] = torch.rand(shape, generator=g, dtype=torch.float64).float() * 0.4 + 0.8
        elif n.endswith("running_var"):
            sd[n] = torch.rand(shape, generator=g, dtype=torch.float64).float() * 0.5 + 0.75
        else:
            sd[n] = torch.randn(shape, generator=g, dtype=torch.float64).float() * 0.1
    return sd


def main():
    assert REF and os.path.isdir(REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_ref_heads as mh

    mh.STUB_TOPLEVEL.update({"torchvision"})
    sys.meta_path.insert(0, mh.StubFinder())
    sys.path.insert(0, REF)
    from det.yolox.models.yolo_head import YOLOXHead
    from det.yolox.models.yolo_pafpn import YOLOPAFPN
    from det.yolox.models.yolox import YOLOX

    m = YOLOX(YOLOPAFPN(depth=DEPTH, width=WIDTH), YOLOXHead(NC, width=WIDTH)).eval()
    names = list(m.state_dict().keys())
    shapes = [",".join(str(d) for d in v.shape) for v in m.state_dict().values()]
    m.load_state_dict(draw_state_dict(names, shapes))
    x = torch.rand(2, 3, 64, 96, generator=torch.Generator().manual_seed(2)) * 255
    with torch.no_grad():
        out = m(x)["det_preds"]
    path = os.path.join(ROOT, "tests", "golden", "ref_yolox.npz")
    np.savez_compressed(path, depth=np.float64(DEPTH), width=np.float64(WIDTH), num_classes=np.int64(NC),
                        names=np.array(names), shapes=np.array(shapes), x=x.numpy(), det_preds=out.numpy())
    print("wrote", path, os.path.getsize(path), "bytes", tuple(out.shape))


if __name__ == "__main__":
    main()
