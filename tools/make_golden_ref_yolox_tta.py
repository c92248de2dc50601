"""Generate tests/golden/ref_yolox_tta.npz by running the REFERENCE's own multi-scale test-time augmentation,
YOLOX.forward(augment=True, cfg) with the scales every shipped BOP test config sets (det/yolox/models/yolox.py:53-86 and
model_utils.scale_img, imported read-only from the checkout that GDRN_REFERENCE_SRC names, with the import stubs of
make_golden_ref_heads.py).

Same model, weights and input as make_golden_ref_yolox.py: depth 0.33, width 0.25, 3 classes, ``draw_state_dict`` (seed
1), input 2 x 3 x 64 x 96 (seed 2).  At 64 x 96 the scales (1, 0.75, 0.83, 1.12, 1.25) give network inputs of 64 x 96
(scale 1, and 0.75 / 0.83 with contents 48 x 72 and 53 x 79) and 96 x 128 (1.12 / 1.25 with contents 71 x 107 and
80 x 120): 882 anchors in all.  Stores the input, det_preds, the scales and the state-dict names / shapes.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_ref_yolox_tta.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_ref_yolox import DEPTH, NC, WIDTH, draw_state_dict  # noqa: E402

SCALES = (1, 0.75, 0.83, 1.12, 1.25)


def main():
    assert REF and os.path.isdir(REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
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
        out = m(x, augment=True, cfg=SimpleNamespace(scales=SCALES))["det_preds"]
    path = os.path.join(ROOT, "tests", "golden", "ref_yolox_tta.npz")
    np.savez_compressed(path, depth=np.float64(DEPTH), width=np.float64(WIDTH), num_classes=np.int64(NC),
                        scales=np.array(SCALES, np.float64), names=np.array(names), shapes=np.array(shapes), x=x.numpy(),
                        det_preds=out.numpy())
    print("wrote", path, os.path.getsize(path), "bytes", tuple(out.shape))


if __name__ == "__main__":
    main()
