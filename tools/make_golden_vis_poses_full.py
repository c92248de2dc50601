"""Generate tests/golden/ref_vis_poses_full.npz by running the REFERENCE's own get_edge and mask2bbox_xyxy
(lib/utils/mask_utils.py) and vis_image_bboxes_cv2 (lib/vis_utils/image.py), imported read-only from the checkout that
GDRN_REFERENCE_SRC names, on seeded synthetic inputs:

  * masks [k,H,W] u8 0/1: ellipses with holes, single-pixel specks, thin lines, masks touching each border, a full
    mask, an empty one and one narrower than bw; -> edges_bw{1,3} [k,H,W] (get_edge(mask, bw, out_channel=1) != 0) and
    bbox_xyxy [k,4] (mask2bbox_xyxy, -1 for the empty mask);
  * a random BGR image and xyxy float boxes (some partly outside the image, some negative) with labels; -> boxed, the
    image vis_image_bboxes_cv2(img, boxes, labels) returns.

Third-party imports the reference makes but which are absent here are stubbed as in make_golden_ref_heads.py; cv2 is
the real one, and mmcv.color_val is restated (a colour name -> its BGR tuple, a tuple as given).

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_vis_poses_full.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_ref_heads as H  # noqa: E402

OUT = os.path.join(H.ROOT, "tests", "golden", "ref_vis_poses_full.npz")
IM_H, IM_W = 40, 56
MMCV_COLORS = {"red": (0, 0, 255), "green": (0, 255, 0), "blue": (255, 0, 0), "cyan": (255, 255, 0),
               "yellow": (0, 255, 255), "magenta": (255, 0, 255), "white": (255, 255, 255), "black": (0, 0, 0)}


def color_val(c):
    return MMCV_COLORS[c] if isinstance(c, str) else tuple(int(v) for v in c)


def masks(rs):
    yy, xx = np.mgrid[0:IM_H, 0:IM_W]
    out = []
    for _ in range(4):   # ellipses with holes and specks
        cx, cy, rx, ry = rs.uniform(8, IM_W - 8), rs.uniform(8, IM_H - 8), rs.uniform(3, 14), rs.uniform(3, 12)
        m = ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1
        m &= rs.rand(IM_H, IM_W) > 0.08
        m |= rs.rand(IM_H, IM_W) > 0.985
        out.append(m)
    for side in range(4):   # touching the top, bottom, left, right border
        m = np.zeros((IM_H, IM_W), bool)
        if side == 0:
            m[:7, 10:30] = True
        elif side == 1:
            m[-5:, 5:50] = True
        elif side == 2:
            m[12:30, :4] = True
        else:
            m[3:38, -9:] = True
        m |= rs.rand(IM_H, IM_W) > 0.99
        out.append(m)
    speck = np.zeros((IM_H, IM_W), bool)
    speck[[0, 5, IM_H - 1, 20], [0, 9, IM_W - 1, 30]] = True
    line = np.zeros((IM_H, IM_W), bool)
    line[17, 3:50] = True
    line[2:36, 41:43] = True
    out += [speck, line, np.ones((IM_H, IM_W), bool), np.zeros((IM_H, IM_W), bool)]
    return np.stack(out).astype(np.uint8)


def main():
    assert H.REF and os.path.isdir(H.REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    H.STUB_TOPLEVEL.update({"numba", "six", "yaml", "png", "imageio", "mmcv", "scipy"})
    sys.meta_path.insert(0, H.StubFinder())
    sys.path.insert(0, H.REF)
    import matplotlib.pyplot as plt   # a stub; image.py sets rcParams at import

    plt.rcParams = {}
    from lib.utils import mask_utils
    from lib.vis_utils import image as vis_image

    vis_image.color_val = color_val
    rs = np.random.RandomState(2024)
    ms = masks(rs)
    out = {"masks": ms}
    for bw in (1, 3):
        out[f"edges_bw{bw}"] = np.stack([mask_utils.get_edge(m, bw=bw, out_channel=1) != 0 for m in ms])
    out["bbox_xyxy"] = np.array([mask_utils.mask2bbox_xyxy(m) if m.any() else [-1] * 4 for m in ms], np.int64)
    img = rs.randint(0, 256, (120, 160, 3)).astype(np.uint8)
    boxes = []
    for _ in range(6):
        x1, y1 = rs.uniform(-20, 150), rs.uniform(-15, 110)
        boxes.append(np.array([x1, y1, x1 + rs.uniform(0.5, 80), y1 + rs.uniform(0.5, 60)]))
    labels = [str(int(v)) for v in rs.randint(1, 30, len(boxes))]
    out.update(image=img, boxes=np.stack(boxes), labels=np.array(labels),
               boxed=vis_image.vis_image_bboxes_cv2(img, boxes, labels))
    np.savez_compressed(OUT, **out)
    print(OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
