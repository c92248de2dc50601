"""Generate tests/golden/ref_vis_poses.npz by running the REFERENCE's own visualization.vis_object_poses
(lib/pysixd/visualization.py, imported read-only from the checkout that GDRN_REFERENCE_SRC names) on stored renders:

  * the renderer is a stand-in whose render_object returns the stored u8 RGB and f32 depth of the instance (keyed by
    its translation);
  * inout.save_im is intercepted to capture the arrays before JPEG encoding;
  * misc.calc_2d_bbox, which lib/pysixd/misc.py does not define, is gt_info.calc_2d_bbox (the BOP toolkit's form);
  * np.float (removed in NumPy 1.24) is float64 and Pillow's removed font.getsize(txt) is (getbbox(txt)[2],
    getbbox(txt)[3]); droid_sans_mono.ttf is not shipped, so the reference falls back to ImageFont.load_default().

Two 24 x 32 images, each run in both resolve modes.  Image 0: three overlapping instances (two at exactly equal
depth), one that renders empty and one cut by the image border; its sensor depth has holes and differs from the renders
on both sides of 15 mm.  Image 1: two instances over a sensor depth with no valid pixel under one of them.
Third-party imports the reference makes but which are absent here are stubbed as in make_golden_ref_heads.py.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_vis_poses.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_ref_heads as H  # noqa: E402

sys.path.insert(0, H.ROOT)
from gdrnpp_bop2022_b200 import gt_info  # noqa: E402

OUT = os.path.join(H.ROOT, "tests", "golden", "ref_vis_poses.npz")
IM_H, IM_W = 24, 32


class StoredRenderer:
    """renderer_py surface: render_object(obj_id, R, t, fx, fy, cx, cy) -> {'rgb', 'depth'} of the stored instance
    whose translation is t."""

    def __init__(self, rgbs, depths, ts):
        self.by_t = {tuple(np.asarray(t, np.float64).ravel()): (r, d) for r, d, t in zip(rgbs, depths, ts)}

    def render_object(self, obj_id, R, t, fx, fy, cx, cy):
        r, d = self.by_t[tuple(np.asarray(t, np.float64).ravel())]
        return {"rgb": r.copy(), "depth": d.copy()}


def blob(rs, cx, cy, rx, ry, z0, sx, sy, color):
    """A tilted elliptic surface (float z, 0 = background) and its flat-shaded-looking u8 render."""
    yy, xx = np.mgrid[0:IM_H, 0:IM_W]
    on = ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1
    d = (z0 + sx * (xx - cx) + sy * (yy - cy) + rs.rand(IM_H, IM_W) * 2).astype(np.float32)
    d[~on] = 0
    shade = 0.5 + 0.5 * rs.rand(IM_H, IM_W)
    rgb = np.round(shade[..., None] * np.asarray(color)[None, None] * 255).astype(np.uint8)
    rgb[~on] = 0
    return rgb, d


def cases(rs):
    """-> [(rgb [H,W,3] u8, depth [H,W] f32 mm, [(m_rgb, m_depth, obj_id)])]."""
    a = blob(rs, 12, 10, 7, 6, 700, 1.0, -0.5, (0.89, 0.28, 0.13))
    b = blob(rs, 17, 12, 6, 5, 690, 0.0, 0.0, (0.45, 0.38, 0.92))
    c = (b[0] // 2 + 40 * (b[0] > 0).astype(np.uint8), b[1].copy())   # exactly b's depth, another colour
    c[0][:, :14] = 0
    c[1][:, :14] = 0
    empty = (np.zeros((IM_H, IM_W, 3), np.uint8), np.zeros((IM_H, IM_W), np.float32))
    edge = blob(rs, 30, 21, 6, 6, 800, -0.4, 0.3, (0.35, 0.73, 0.63))
    im0 = [(a[0], a[1], 1), (b[0], b[1], 2), (c[0], c[1], 3), (empty[0], empty[1], 4), (edge[0], edge[1], 5)]
    d = blob(rs, 8, 8, 6, 6, 900, 0.5, 0.5, (0.62, 0.28, 0.91))
    e = blob(rs, 22, 16, 7, 5, 640, -0.3, 0.2, (0.65, 0.71, 0.22))
    im1 = [(d[0], d[1], 1), (e[0], e[1], 2)]
    out = []
    for k, inst in enumerate((im0, im1)):
        rgb = (rs.rand(IM_H, IM_W, 3) * 255).astype(np.uint8)
        depth = np.full((IM_H, IM_W), 1000.0, np.float32)
        for _, md, _ in inst[::-1]:
            on = md > 0
            depth[on] = md[on]
        depth = (depth + rs.randn(IM_H, IM_W).astype(np.float32) * 12).astype(np.float32)   # both sides of 15 mm
        if k == 0:
            depth[3:7, 4:9] = 0        # holes
            depth[12:15, 10:20] -= 40  # the renders lie behind the sensor by more than 15 mm here
        else:
            depth[:, :16] = 0          # no sensor depth under instance d
        out.append((rgb, depth, inst))
    return out


def main():
    assert H.REF and os.path.isdir(H.REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    H.STUB_TOPLEVEL.update({"cv2", "numba", "six", "yaml", "png", "imageio", "mmcv", "scipy"})
    sys.meta_path.insert(0, H.StubFinder())
    sys.path.insert(0, H.REF)
    np.float = np.float64
    from PIL import ImageFont

    for cls in (ImageFont.FreeTypeFont, ImageFont.ImageFont):
        cls.getsize = lambda self, txt: tuple(self.getbbox(txt)[2:4])
    from lib.pysixd import inout, misc, visualization

    misc.calc_2d_bbox = lambda xs, ys, im_size: gt_info.calc_2d_bbox(xs, ys)
    misc.ensure_dir = lambda path: None
    misc.log = lambda *a, **k: None
    saved = {}
    inout.save_im = lambda path, im, jpg_quality=95: saved.__setitem__(path, np.array(im))
    rs = np.random.RandomState(2026)
    K = np.array([[40.0, 0, 15.3], [0, 41.0, 11.7], [0, 0, 1]])
    out = {"K": K}
    for i, (rgb, depth, inst) in enumerate(cases(rs)):
        ts = [np.array([[0.0], [0.0], [1000.0 + k]]) for k in range(len(inst))]
        ren = StoredRenderer([m[0] for m in inst], [m[1] for m in inst], ts)
        poses = [{"obj_id": o, "R": np.eye(3), "t": t, "text_info": [{"name": "", "val": "{}:{}".format(o, k), "fmt": ""}]}
                 for k, ((_, _, o), t) in enumerate(zip(inst, ts))]
        out[f"im{i}_rgb"], out[f"im{i}_depth"] = rgb, depth
        out[f"im{i}_m_rgb"] = np.stack([m[0] for m in inst])
        out[f"im{i}_m_depth"] = np.stack([m[1] for m in inst])
        out[f"im{i}_obj_ids"] = np.array([m[2] for m in inst])
        for resolve in (True, False):
            saved.clear()
            visualization.vis_object_poses(poses, K, ren, rgb=rgb, depth=depth, vis_rgb_path="rgb",
                                           vis_depth_diff_path="diff", vis_rgb_resolve_visib=resolve)
            out[f"im{i}_resolve{int(resolve)}_vis_rgb"] = saved["rgb"]
            out[f"im{i}_resolve{int(resolve)}_vis_depth_diff"] = saved["diff"]
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
