"""Generate tests/golden/ref_gt_info.npz by running the REFERENCE's own GT-annotation code (imported read-only from the
checkout that GDRN_REFERENCE_SRC names) on stored depth maps:

  * the per-instance loop of lib/pysixd/scripts/calc_gt_info.py:110-173 and of calc_gt_masks.py:92-111, read from the
    scripts' source and executed as they stand, with the reference's misc.depth_im_to_dist_im_fast and
    visibility.estimate_visib_mask_gt.  The renderer is a stand-in whose render_object returns the stored float depth
    of the instance: a 3x-canvas render for calc_gt_info.py and an image-size render for calc_gt_masks.py.
  * misc.calc_2d_bbox, which the script calls but lib/pysixd/misc.py does not define, is supplied as
    gdrnpp_bop2022_b200.gt_info.calc_2d_bbox (the BOP toolkit's definition).
  * inout.save_json of one scene_gt_info dict, stored as bytes.

Two images (different K and depth_scale); their sensor depth has holes, an occluder, and instances cut by the image
border, fully outside it, fully occluded, empty, and over missing depth.  Third-party imports the reference makes but
which are absent here are stubbed exactly as in make_golden_ref_heads.py.

  GDRN_REFERENCE_SRC=<reference checkout> python tools/make_golden_gt_info.py
"""
import json
import os
import sys
import tempfile
import textwrap

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_ref_heads as H  # noqa: E402

sys.path.insert(0, H.ROOT)
from gdrnpp_bop2022_b200 import gt_info  # noqa: E402

OUT = os.path.join(H.ROOT, "tests", "golden", "ref_gt_info.npz")
IM_H, IM_W = 24, 32
DELTA = 15


def script_lines(name, first, last, indent):
    """Lines first..last (1-based, inclusive) of a reference script, dedented by `indent` spaces."""
    with open(os.path.join(H.REF, "lib", "pysixd", "scripts", name)) as f:
        lines = f.read().split("\n")[first - 1:last]
    return textwrap.dedent("\n".join(l[indent:] if l.strip() else "" for l in lines))


class StoredDepthRenderer:
    """renderer_type 'python' surface: render_object(obj_id, R, t, fx, fy, cx, cy) -> {'depth'}, the stored depth of
    the instance whose translation is t."""

    def __init__(self, depths, gts):
        self.by_t = {tuple(np.asarray(g["cam_t_m2c"], np.float64).ravel()): d for g, d in zip(gts, depths)}

    def render_object(self, obj_id, R, t, fx, fy, cx, cy):
        return {"depth": self.by_t[tuple(np.asarray(t, np.float64).ravel())]}


def blob(rs, cx, cy, rx, ry, z0, sx, sy):
    """A tilted elliptic surface on the 3x canvas (float z, 0 = background), centre (cx, cy) in canvas pixels."""
    yy, xx = np.mgrid[0:3 * IM_H, 0:3 * IM_W]
    d = (z0 + sx * (xx - cx) + sy * (yy - cy) + rs.rand(3 * IM_H, 3 * IM_W) * 2).astype(np.float32)
    d[((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 > 1] = 0
    return d


def cases(rs):
    """-> (images [(K, depth_scale, sensor u16 [H,W])], instances [(image, canvas render [3H,3W])])."""
    W, Hh = IM_W, IM_H
    inst = [
        (0, blob(rs, W + 16, Hh + 12, 9, 7, 700, 1.2, -0.8)),      # inside, partly occluded, over holes
        (0, blob(rs, W + 2, Hh + 20, 8, 8, 650, -0.5, 0.3)),       # cut by the left and bottom border
        (0, blob(rs, W - 15, Hh - 12, 6, 5, 720, 0.0, 0.0)),       # fully outside the image: -1 boxes
        (0, blob(rs, W + 26, Hh + 5, 4, 4, 900, 0.2, 0.2)),        # fully occluded
        (0, np.zeros((3 * Hh, 3 * W), np.float32)),                # nothing rendered
        (1, blob(rs, W + 10, Hh + 10, 10, 8, 800, 0.7, 0.4)),      # over missing sensor depth: visible under bop19
        (1, blob(rs, 2 * W - 3, 2 * Hh - 3, 12, 12, 760, -0.3, 0.6)),   # cut by the right and bottom border
    ]
    images = []
    for i, (K, scale) in enumerate(((np.array([[40.0, 0, 15.3], [0, 41.0, 11.7], [0, 0, 1]]), 0.1),
                                    (np.array([[37.5, 0, 16.6], [0, 36.25, 12.2], [0, 0, 1]]), 1.0))):
        mm = np.full((Hh, W), 1000.0) + rs.rand(Hh, W) * 3
        for img, d in inst:
            win = d[Hh:2 * Hh, W:2 * W]
            if img == i:
                on = win > 0
                mm[on] = win[on] + rs.randn(int(on.sum())) * 6    # the surface itself, within a few mm
        if i == 0:
            mm[7:11, 8:12] = 0                                     # holes
            mm[12:18, 14:20] = 520                                 # occluder in front of instance 0
            mm[0:11, 21:32] = 480                                  # covers instance 3 entirely
        else:
            mm[2:20, 0:22] = 0                                     # no depth over instance 5
        images.append((K, scale, np.round(mm / scale).astype(np.uint16)))
    return images, inst


def main():
    assert H.REF and os.path.isdir(H.REF), "set GDRN_REFERENCE_SRC to a checkout of the reference project"
    H.STUB_TOPLEVEL.update({"cv2", "numba", "six", "yaml", "png", "imageio"})
    sys.meta_path.insert(0, H.StubFinder())
    sys.path.insert(0, H.REF)
    for _n, _v in (("float", float), ("int", int), ("bool", bool)):
        if not hasattr(np, _n):
            setattr(np, _n, _v)
    from lib.pysixd import inout, misc, visibility

    misc.calc_2d_bbox = lambda xs, ys, im_size: gt_info.calc_2d_bbox(xs, ys)
    rs = np.random.RandomState(2023)
    images, inst = cases(rs)
    info_body = script_lines("calc_gt_info.py", 110, 173, 8)
    masks_body = script_lines("calc_gt_masks.py", 92, 111, 8)
    infos, masks, masks_visib, depth_img = {}, [], [], []
    for i, (K, scale, sensor) in enumerate(images):
        idx = [k for k, (img, _) in enumerate(inst) if img == i]
        gts = [{"obj_id": 1, "cam_R_m2c": np.eye(3), "cam_t_m2c": np.array([[0.0], [0.0], [1000.0 + k]])} for k in idx]
        large = [inst[k][1] for k in idx]
        small = []
        for k, d in zip(idx, large):
            s = d[IM_H:2 * IM_H, IM_W:2 * IM_W].copy()
            if k == 0:   # the image-size render is a render of its own, not the canvas window
                s[s > 0] += np.float32(3.0)
                s[IM_H // 2, :] = 0
            small.append(s)
        depth_img += small
        # calc_gt_info.py:96-107 (inout.load_depth is imread(...).astype(np.float32)), then the per-instance loop
        depth = sensor.astype(np.float32)
        depth *= scale
        fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
        ns = {"np": np, "misc": misc, "visibility": visibility, "p": {"delta": DELTA, "vis_visibility_masks": False},
              "ren": StoredDepthRenderer(large, gts), "scene_gt": {i: gts}, "im_id": i, "scene_gt_info": {i: []},
              "K": K, "fx": fx, "fy": fy, "cx": cx, "cy": cy, "depth": depth, "im_size": (IM_W, IM_H),
              "ren_cx_offset": IM_W, "ren_cy_offset": IM_H, "im_width": IM_W, "im_height": IM_H}
        exec(info_body, ns)
        infos[i] = ns["scene_gt_info"][i]
        # calc_gt_masks.py:83-90, then the per-instance loop with inout.save_im capturing the arrays
        saved = {}
        stub_inout = type("inout", (), {"save_im": staticmethod(lambda path, im: saved.__setitem__(path, im))})
        dp_split = {"mask_tpath": "mask/{scene_id}_{im_id}_{gt_id}", "mask_visib_tpath": "visib/{scene_id}_{im_id}_{gt_id}"}
        ns = {"np": np, "misc": misc, "visibility": visibility, "inout": stub_inout, "p": {"delta": DELTA},
              "ren": StoredDepthRenderer(small, gts), "scene_gt": {i: gts}, "im_id": i, "scene_id": 0, "dp_split": dp_split,
              "fx": fx, "fy": fy, "cx": cx, "cy": cy, "K": K, "dist_im": misc.depth_im_to_dist_im_fast(depth, K)}
        exec(masks_body, ns)
        for g in range(len(idx)):
            masks.append(saved["mask/0_{}_{}".format(i, g)])
            masks_visib.append(saved["visib/0_{}_{}".format(i, g)])
    recs = [r for i in sorted(infos) for r in infos[i]]
    out = {
        "K": np.stack([im[0] for im in images]), "depth_scale": np.array([im[1] for im in images]),
        "depth_test": np.stack([im[2] for im in images]), "inst_img": np.array([img for img, _ in inst], np.int32),
        "depth_large": np.stack([d for _, d in inst]), "depth_img": np.stack(depth_img), "delta": np.array(float(DELTA)),
        "mask": np.stack(masks), "mask_visib": np.stack(masks_visib),
        "px_count_all": np.array([r["px_count_all"] for r in recs]),
        "px_count_valid": np.array([r["px_count_valid"] for r in recs]),
        "px_count_visib": np.array([r["px_count_visib"] for r in recs]),
        "visib_fract": np.array([r["visib_fract"] for r in recs]),
        "bbox_obj": np.array([r["bbox_obj"] for r in recs]), "bbox_visib": np.array([r["bbox_visib"] for r in recs]),
    }
    # inout.save_json of a scene_gt_info dict: images out of order, one without instances
    scene_info = {5: infos[1], 2: [], 0: infos[0]}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "scene_gt_info.json")
        inout.save_json(path, {k: scene_info[k] for k in sorted(scene_info)})
        with open(path, "rb") as f:
            out["save_json_bytes"] = np.frombuffer(f.read(), np.uint8)
    out["save_json_content"] = np.frombuffer(json.dumps({str(k): v for k, v in scene_info.items()}).encode(), np.uint8)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")
    for r in recs:
        print(r)


if __name__ == "__main__":
    main()
