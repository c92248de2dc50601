"""Pose visualisation of a BOP split on the GPU: the reference's vis_gt_poses.py without a GL context.

Mirrors lib/pysixd/scripts/vis_gt_poses.py and visualization.vis_object_poses (lib/pysixd/visualization.py:93-260):
per image, every instance is rendered flat-shaded in a uniform colour (renderer.render_meshes_rgb, one launch for the
instances of many images), then one composite pass (csrc/vis_poses.cu) resolves visibility, blends with the image,
finds each instance's box and forms the depth-difference image.  Only the PIL rectangles and text are drawn on the host,
on a sparse info layer added with saturation; JPEG writes go to a writer pool.

  python -m gdrnpp_bop2022_b200.vis_poses --dataset lmo --dataset_split test
  python -m gdrnpp_bop2022_b200.vis_poses --dataset lmo --dataset_split test --result_filename gdrn_lmo-test.csv
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

if __package__ in (None, ""):   # run by path
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    __package__ = "gdrnpp_bop2022_b200"

import numpy as np
import torch

from . import _lib
from . import bop_eval
from . import gt_info
from ._lib import GdrnError

DEFAULT_MAX_BYTES = 2 << 30
RGB, RESOLVE, DEPTH_DIFF = 1, 2, 4
DELTA = 15
JPEG_QUALITY = 95


# ---------------------------------------------------------------------------------------------------------------------
# Host drawing: visualization.draw_rect / write_text_on_image / depth_for_vis, restated for NumPy 2 and Pillow >= 10
def font():
    """The reference's font: droid_sans_mono.ttf is not shipped with it, so its fallback ImageFont.load_default()."""
    from PIL import ImageFont

    global _FONT
    if _FONT is None:
        _FONT = ImageFont.load_default()
    return _FONT


_FONT = None


def _draw_text(draw, txt_list, loc, color):
    """write_text_on_image's loop on a PIL draw: one line per entry, the line height getbbox(txt)[3] (Pillow 10
    removed the reference's font.getsize, whose height this is)."""
    f = font()
    for info in txt_list:
        tpl = ("{}:{" if info["name"] != "" else "{}{") + info["fmt"] + "}"
        txt = tpl.format(info["name"], info["val"])
        draw.text(loc, txt, fill=tuple(int(c * 255) for c in color), font=f)
        loc = (loc[0], loc[1] + f.getbbox(txt)[3])


def write_text_on_image(im, txt_list, loc=(3, 0), color=(1.0, 1.0, 1.0)):
    """visualization.write_text_on_image (u8 [H,W,3] -> new array)."""
    from PIL import Image, ImageDraw

    pil = Image.fromarray(im)
    _draw_text(ImageDraw.Draw(pil), txt_list, loc, color)
    return np.array(pil)


def info_layer(H, W, boxes, texts):
    """The black info layer of vis_object_poses: per instance with a box (x, y, w, h), draw_rect in 0.3 grey, then its
    text in white at (x + 2, y).  -> (layer u8 [h,w,3], (x0, y0)) cropped to what was drawn, or None."""
    from PIL import Image, ImageDraw

    if not boxes:
        return None
    pil = Image.new("RGB", (W, H))
    draw = ImageDraw.Draw(pil)
    for (x, y, w, h), txt in zip(boxes, texts):
        draw.rectangle((x, y, x + w, y + h), outline=tuple(int(c * 255) for c in (0.3, 0.3, 0.3)), fill=None)
        if txt is not None:
            _draw_text(draw, txt, (x + 2, y), (1.0, 1.0, 1.0))
    bb = pil.getbbox()
    if bb is None:
        return None
    return np.asarray(pil.crop(bb)), (bb[0], bb[1])


def add_layer(blend, layer):
    """blend + layer with saturation at 255, in place, over the layer's crop."""
    if layer is None:
        return blend
    im, (x0, y0) = layer
    h, w = im.shape[:2]
    win = blend[y0:y0 + h, x0:x0 + w]
    win[...] = np.minimum(win.astype(np.uint16) + im, 255).astype(np.uint8)
    return blend


def depth_diff_text(vmin, vmax, vmean):
    return [{"name": "min diff", "fmt": ":.3f", "val": vmin}, {"name": "max diff", "fmt": ":.3f", "val": vmax},
            {"name": "mean diff", "fmt": ":.3f", "val": vmean}]


def draw_depth_diff_text(vis, txt_list):
    """write_text_on_image(depth_diff_vis, depth_info) at (3, 0), drawn on the crop the text covers only."""
    from PIL import Image, ImageDraw

    f = font()
    x1 = y1 = 0
    y = 0
    for info in txt_list:
        tpl = ("{}:{" if info["name"] != "" else "{}{") + info["fmt"] + "}"
        bb = f.getbbox(tpl.format(info["name"], info["val"]))
        x1, y1 = max(x1, 3 + bb[2] + 1), max(y1, y + bb[3] + 1)
        y += bb[3]
    x1, y1 = min(x1, vis.shape[1]), min(y1, vis.shape[0])
    pil = Image.fromarray(np.ascontiguousarray(vis[:y1, :x1]))
    _draw_text(ImageDraw.Draw(pil), txt_list, (3, 0), (1.0, 1.0, 1.0))
    vis[:y1, :x1] = np.asarray(pil)
    return vis


def depth_for_vis(depth, valid_start=0.2, valid_end=1.0):
    """visualization.depth_for_vis in f64 (np.float is float64).  The reference raises on an empty mask and makes NaN
    when every masked value is equal; here those give 0 and valid_start."""
    mask = depth > 0
    out = depth.astype(np.float64)
    if not mask.any():
        return out
    out[mask] -= out[mask].min()
    mx = out[mask].max()
    if mx == 0:
        out[mask] = 0.0
    else:
        out[mask] /= mx / (valid_end - valid_start)
    out[mask] += valid_start
    return out


def host_vis_object_poses(m_rgb, m_depth, rgb, depth, texts, resolve_visib=True, rgb_vis=True, depth_diff=True):
    """The NumPy arithmetic of visualization.vis_object_poses for one image, from its instance renders m_rgb [k,H,W,3]
    u8 and m_depth [k,H,W] f32: the reference the kernel is tested against and the host arm of bench_vis_poses.py (the
    product path never calls it).  texts: per instance the text_info list or None.
    -> {"rgb": u8 [H,W,3] (with rgb_vis), "depth_diff": u8 [H,W,3] (with depth_diff), "boxes": [(x, y, w, h) | None]}."""
    H, W = (rgb if rgb is not None else depth).shape[:2]
    ren_rgb = np.zeros((H, W, 3), np.uint8)
    ren_depth = np.zeros((H, W), np.float32)
    need_depth = depth_diff or (rgb_vis and resolve_visib)
    boxes = []
    for k in range(len(m_depth if m_depth is not None else m_rgb)):
        m_mask = None
        if need_depth:
            md = m_depth[k]
            m_mask = np.logical_and(md != 0, np.logical_or(ren_depth == 0, md < ren_depth))
            ren_depth[m_mask] = md[m_mask]
        if rgb_vis:
            mr = m_rgb[k]
            if resolve_visib:
                ren_rgb[m_mask] = mr[m_mask]
            else:
                f = ren_rgb.astype(np.float32) + mr.astype(np.float32)
                f[f > 255] = 255
                ren_rgb = f.astype(np.uint8)
            ys, xs = np.sum(mr > 0, axis=2).nonzero()
            boxes.append(gt_info.calc_2d_bbox(xs, ys) if len(ys) else None)
    out = {"boxes": boxes}
    if rgb_vis:
        drawn = [(b, t) for b, t in zip(boxes, texts) if b is not None]
        layer = np.zeros((H, W, 3), np.uint8)
        if drawn:
            from PIL import Image, ImageDraw

            pil = Image.fromarray(layer)
            draw = ImageDraw.Draw(pil)
            for (x, y, w, h), t in drawn:
                draw.rectangle((x, y, x + w, y + h), outline=(76, 76, 76), fill=None)
                if t is not None:
                    _draw_text(draw, t, (x + 2, y), (1.0, 1.0, 1.0))
            layer = np.asarray(pil)
        v = 0.5 * rgb.astype(np.float32) + 0.5 * ren_rgb.astype(np.float32) + 1.0 * layer.astype(np.float32)
        v[v > 255] = 255
        out["rgb"] = v.astype(np.uint8)
    if depth_diff:
        valid = (depth > 0) * (ren_depth > 0)
        diff = valid * (ren_depth.astype(np.float32) - depth)
        below = (255 * (valid * (diff < DELTA))).astype(np.uint8)
        gb = 255 * depth_for_vis(diff - diff.min())
        vis = np.dstack([below, gb, gb]).astype(np.uint8)
        vis[np.logical_not(valid)] = 0
        dv = diff[valid]
        if dv.size:
            vis = write_text_on_image(vis, depth_diff_text(np.min(dv), np.max(dv), np.mean(dv)))
        out["depth_diff"] = vis
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Device passes
def composite_device(m_rgb, m_depth, inst_off, rgb, depth, flags, inst_off_dev=None):
    """One gdrn_vis_poses launch set over N images of one size.  m_rgb [n,H,W,3] u8, m_depth [n,H,W] f32, inst_off
    [N+1] host array (image j owns instances inst_off[j]:inst_off[j+1]), rgb [N,H,W,3] u8, depth [N,H,W] f32 mm, all on
    one CUDA device; inst_off_dev: inst_off already on that device as int32 (saves one copy per call).
    -> dict of device tensors (see include/gdrn_b200.h); no synchronisation."""
    dev = depth.device if depth is not None else rgb.device
    N, H, W = (int(s) for s in (depth if depth is not None else rgb).shape[:3])
    off_h = np.asarray(inst_off, np.int64)
    n, max_inst = int(off_h[-1]), int(np.diff(off_h).max())
    off = inst_off_dev if inst_off_dev is not None else torch.from_numpy(off_h.astype(np.int32)).to(dev)
    do_rgb, do_diff = bool(flags & RGB), bool(flags & DEPTH_DIFF)
    need_depth = do_diff or (do_rgb and flags & RESOLVE)
    e = lambda shape, dt, on: torch.empty(shape, dtype=dt, device=dev) if on else None   # noqa: E731
    res = {"ren_rgb": e((N, H, W, 3), torch.uint8, do_rgb), "blend": e((N, H, W, 3), torch.uint8, do_rgb),
           "boxes": e((max(n, 1), 4), torch.int32, do_rgb), "ren_depth": e((N, H, W), torch.float32, need_depth),
           "diff_vis": e((N, H, W, 3), torch.uint8, do_diff), "diff_minmax": e((N, 2), torch.float32, do_diff),
           "diff_sum": e((N,), torch.float64, do_diff), "diff_count": e((N,), torch.int64, do_diff)}
    L = _lib.lib()
    wsb = L.gdrn_vis_poses_workspace_bytes(N, H, W)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.gdrn_vis_poses(_lib.ptr(m_rgb if do_rgb else None), _lib.ptr(m_depth if need_depth else None),
                                    _lib.ptr(off), max_inst, N, n, _lib.ptr(rgb if do_rgb else None),
                                    _lib.ptr(depth if do_diff else None), H, W, int(flags), _lib.ptr(res["ren_rgb"]),
                                    _lib.ptr(res["ren_depth"]), _lib.ptr(res["blend"]), _lib.ptr(res["boxes"]),
                                    _lib.ptr(res["diff_vis"]), _lib.ptr(res["diff_minmax"]), _lib.ptr(res["diff_sum"]),
                                    _lib.ptr(res["diff_count"]), _lib.ptr(ws), wsb, _lib.current_stream()),
                   "gdrn_vis_poses")
    if do_rgb:
        res["boxes"] = res["boxes"][:n]
    return res


def finish_host(res, inst_off, texts, flags):
    """Host side of one composite: the info layers and the depth-difference text.  res: the composite's outputs as
    host arrays.  -> [{"rgb", "depth_diff"} per image]."""
    N = len(inst_off) - 1
    out = []
    for j in range(N):
        o = {}
        if flags & RGB:
            b = res["boxes"][inst_off[j]:inst_off[j + 1]]
            keep = [k for k in range(len(b)) if b[k, 0] <= b[k, 2]]
            boxes = [(int(b[k, 0]), int(b[k, 1]), int(b[k, 2] - b[k, 0]), int(b[k, 3] - b[k, 1])) for k in keep]
            t = texts[j]
            blend = res["blend"][j].copy()
            H, W = blend.shape[:2]
            o["rgb"] = add_layer(blend, info_layer(H, W, boxes, [t[k] for k in keep]))
        if flags & DEPTH_DIFF:
            vis = res["diff_vis"][j].copy()
            cnt = int(res["diff_count"][j])
            if cnt:   # np.float32 values, formatted as the reference formats np.min / np.max / np.mean of f32
                vis = draw_depth_diff_text(vis, depth_diff_text(np.float32(res["diff_minmax"][j, 0]),
                                                                np.float32(res["diff_minmax"][j, 1]),
                                                                np.float32(res["diff_sum"][j] / cnt)))
            o["depth_diff"] = vis
        out.append(o)
    return out


def _flags(resolve_visib, rgb_vis, depth_diff):
    if not (rgb_vis or depth_diff):
        raise GdrnError("vis_poses: nothing to visualise (rgb_vis and depth_diff both off)")
    return (RGB if rgb_vis else 0) | (RESOLVE if resolve_visib else 0) | (DEPTH_DIFF if depth_diff else 0)


def render_instances(meshes, poses_per_image, K, H, W, obj_colors=None):
    """Flat-shaded renders of every instance of every image, one launch: poses_per_image[j] = [{obj_id, R, t}], K
    [N,3,3] (mm).  obj_colors: {obj_id: (r, g, b)} uniform surface colours, or None for the meshes' own colours.
    -> (m_rgb [n,H,W,3] u8, m_depth [n,H,W] f32, inst_off [N+1]) on the meshes' device."""
    from . import renderer

    inst = [(j, p) for j, ps in enumerate(poses_per_image) for p in ps]
    inst_off = np.cumsum([0] + [len(ps) for ps in poses_per_image]).astype(np.int64)
    n, dev = len(inst), meshes.device
    if n == 0:
        return None, None, inst_off
    try:
        ids = torch.tensor([meshes.ids[int(p["obj_id"])] for _, p in inst], dtype=torch.int32, device=dev)
    except KeyError as e:
        raise GdrnError(f"vis_poses: no model for obj_id {e.args[0]}") from None
    poses = np.concatenate([np.stack([np.asarray(p["R"], np.float64).reshape(3, 3) for _, p in inst]),
                            np.stack([np.asarray(p["t"], np.float64).reshape(3, 1) for _, p in inst])], axis=2)
    Ks = np.asarray(K, np.float64).reshape(-1, 3, 3)[[j for j, _ in inst]]
    cols = None
    if obj_colors is not None:
        try:
            cols = torch.tensor([obj_colors[int(p["obj_id"])] for _, p in inst], dtype=torch.float32)
        except KeyError as e:
            raise GdrnError(f"vis_poses: no colour for obj_id {e.args[0]}") from None
    rgb, depth = renderer.render_meshes_rgb(ids, torch.from_numpy(poses).to(dev), torch.from_numpy(Ks).to(dev), H, W,
                                            bop_eval.VSD_ZNEAR, bop_eval.VSD_ZFAR, colors=cols)
    return rgb, depth, inst_off


def vis_object_poses(meshes, poses_per_image, K, rgb, depth, resolve_visib=True, rgb_vis=True, depth_diff=True,
                     obj_colors=None):
    """visualization.vis_object_poses for a batch of N images of one size, in memory.  meshes: bop_eval.VsdMeshes (mm);
    poses_per_image[j] = [{obj_id, R [3,3], t [3] mm, text_info (optional)}] in drawing order; K [N,3,3]; rgb [N,H,W,3]
    u8 (with rgb_vis); depth [N,H,W] f32 in mm (with depth_diff or resolve_visib).  obj_colors: {obj_id: (r, g, b)}.
    -> [{"rgb": u8 [H,W,3], "depth_diff": u8 [H,W,3]} per image]: the arrays the reference saves."""
    flags = _flags(resolve_visib, rgb_vis, depth_diff)
    ref = rgb if rgb_vis else depth
    N, H, W = (int(s) for s in np.shape(ref)[:3])
    dev = meshes.device
    with torch.cuda.device(dev):
        m_rgb, m_depth, inst_off = render_instances(meshes, poses_per_image, K, H, W, obj_colors)
        t_rgb = torch.tensor(np.asarray(rgb, np.uint8)).to(dev) if rgb_vis else None
        t_depth = None
        if depth_diff or (rgb_vis and resolve_visib):
            t_depth = torch.tensor(np.asarray(depth, np.float32)).reshape(N, H, W).to(dev)
        res = composite_device(m_rgb, m_depth, inst_off, t_rgb, t_depth, flags)
        host = {k: v.cpu().numpy() for k, v in res.items() if v is not None}
    texts = [[p.get("text_info") for p in ps] for ps in poses_per_image]
    return finish_host(host, inst_off, texts, flags)


# ---------------------------------------------------------------------------------------------------------------------
# Split driver
def default_colors():
    """The uniform colour of obj_id is colors[(obj_id - 1) % len(colors)].  The reference reads
    lib/pysixd/colors.json (pass it with --colors_json); without it, 30 hues evenly spaced around the colour wheel."""
    import colorsys

    return [list(colorsys.hsv_to_rgb((k * 7 % 30) / 30.0, 0.7, 0.9)) for k in range(30)]


def plan_images(sp, scene_ids=None, im_ids=None, gt_ids=None, targets=None, results=None, rgb_vis=True):
    """[(scene_id, im_id, K, depth_scale, depth path, image path, poses)] in the script's order.  GT poses carry text
    "{obj_id}:{gt_id}"; with results ({(scene_id, im_id): [rows in file order]}) the estimates are drawn instead,
    with text "{obj_id}:{score:.2f}".  The image path is resolved (and must exist) only with rgb_vis."""
    scenes = gt_info.plan_split(sp, scene_ids)
    out = []
    for scene_id, ims in scenes:
        sel = None if targets is None else targets.get(scene_id, set())
        for im in ims:
            im_id = im["im_id"]
            if (sel is not None and im_id not in sel) or (im_ids and im_id not in im_ids):
                continue
            if results is not None:
                rows = results.get((scene_id, im_id), [])
                poses = [{"obj_id": r["obj_id"], "R": r["R"], "t": r["t"],
                          "text_info": [{"name": "", "val": "{}:{:.2f}".format(r["obj_id"], r["score"]), "fmt": ""}]}
                         for r in rows]
            else:
                poses = [{"obj_id": int(g["obj_id"]), "R": g["cam_R_m2c"], "t": g["cam_t_m2c"],
                          "text_info": [{"name": "", "val": "{}:{}".format(g["obj_id"], gid), "fmt": ""}]}
                         for gid, g in enumerate(im["gts"]) if not gt_ids or gid in gt_ids]
            out.append((scene_id, im_id, np.asarray(im["K"], np.float64).reshape(3, 3), im["depth_scale"], im["depth"],
                        gt_info.image_path(sp, scene_id, im_id) if rgb_vis else None, poses))
    return out


def read_rgb(path):
    """inout.load_im(path)[:, :, :3] (imageio reads through Pillow); a gray image is stacked three times."""
    from PIL import Image

    a = np.asarray(Image.open(path))
    if a.ndim == 2:
        return np.dstack([a, a, a])
    return np.ascontiguousarray(a[:, :, :3])


def _decode(batch, need_rgb, need_depth):
    """-> (rgb [B,H,W,3] u8 pinned, depth [B,H,W] f32 mm pinned): inout.load_depth(...) * depth_scale in f32."""
    pin = torch.cuda.is_available()
    rgbs = [read_rgb(b[5]) for b in batch] if need_rgb else None
    deps = None
    if need_depth:
        deps = [gt_info.read_depth(b[4]).astype(np.float32) * np.float32(b[3]) for b in batch]
    ref = rgbs[0] if need_rgb else deps[0]
    H, W = ref.shape[:2]
    for k, b in enumerate(batch):
        for a, what in ((rgbs and rgbs[k], b[5]), (deps and deps[k], b[4])):
            if a is not None and a.shape[:2] != (H, W):
                raise GdrnError("image {} is {}x{}, other images of its batch are {}x{}".format(what, a.shape[1],
                                                                                              a.shape[0], W, H))
    r = torch.from_numpy(np.stack(rgbs)).pin_memory() if need_rgb and pin else (
        torch.from_numpy(np.stack(rgbs)) if need_rgb else None)
    d = torch.from_numpy(np.stack(deps)).pin_memory() if need_depth and pin else (
        torch.from_numpy(np.stack(deps)) if need_depth else None)
    return r, d


def _batches(images, max_bytes, need_depth):
    """Consecutive images of one size, at most max_bytes of renders and composites each (the size of the first
    image of the batch is read from its depth or colour file header)."""
    from PIL import Image

    out, cur, cur_bytes, cur_size = [], [], 0, None
    for im in images:
        with Image.open(im[4] if need_depth else im[5]) as f:
            size = f.size
        b = (len(im[6]) * 16 + 24) * size[0] * size[1]
        if cur and (size != cur_size or cur_bytes + b > max_bytes):
            out.append(cur)
            cur, cur_bytes = [], 0
        cur.append(im)
        cur_bytes += b
        cur_size = size
    if cur:
        out.append(cur)
    return out


def _save_jpg(path, im):
    from PIL import Image

    Image.fromarray(im).save(path, quality=JPEG_QUALITY)


def run_split(sp, model_dir, vis_path, dataset, split, scene_ids=None, im_ids=None, gt_ids=None, targets=None,
              results=None, rgb_vis=True, resolve_visib=True, depth_diff=True, colors=None, vis_orig_color=False,
              max_bytes=DEFAULT_MAX_BYTES, workers=8, device="cuda", meshes=None):
    """Visualise every selected image of a split; writes {vis_path}/{dataset}/{split}/{scene:06d}/{im:06d}.jpg and
    {im:06d}_depth_diff.jpg.  -> {"images", "instances", "seconds"}."""
    from .ply import load_ply
    from .renderer import load_texture

    flags = _flags(resolve_visib, rgb_vis, depth_diff)
    need_depth = bool(depth_diff or (rgb_vis and resolve_visib))
    images = plan_images(sp, scene_ids, im_ids, gt_ids, targets, results, rgb_vis)
    used = sorted({int(p["obj_id"]) for im in images for p in im[6]})
    obj_colors = None
    if not vis_orig_color:
        colors = colors or default_colors()
        obj_colors = {o: tuple(colors[(o - 1) % len(colors)]) for o in used}
    if meshes is None:
        models = {}
        for o in used:
            p = os.path.join(model_dir, "obj_{:06d}.ply".format(o))
            if not os.path.exists(p):
                raise GdrnError("obj_id {}: no model file {}".format(o, p))
            m = load_ply(p)
            if "faces" not in m:
                raise GdrnError("obj_id {}: {} has no faces".format(o, p))
            col = uvs = tex = None
            if vis_orig_color:
                # renderer_py.py:340-365: the PLY's texture (comment TextureFile, beside the model) with its per-vertex
                # UVs, else its vertex colours
                if "texture_file" in m:
                    tp = os.path.join(os.path.dirname(p), m["texture_file"])
                    if "texture_uv" not in m:
                        raise GdrnError("obj_id {}: {} is textured; --vis_orig_color needs per-vertex texture_u / "
                                        "texture_v".format(o, p))
                    if not os.path.exists(tp):
                        raise GdrnError("obj_id {}: {} is textured; --vis_orig_color needs its texture {}".format(o, p, tp))
                    uvs, tex = m["texture_uv"], load_texture(tp)
                elif "colors" in m:
                    col = m["colors"] / 255.0 if m["colors"].max() > 1.0 else m["colors"]
            models[o] = (m["pts"], m["faces"], col, uvs, tex)
        meshes = bop_eval.VsdMeshes(models, device=device) if models else None
    batches = _batches(images, max_bytes, need_depth)
    decode_pool, write_pool = ThreadPoolExecutor(max(1, workers)), ThreadPoolExecutor(max(1, workers))
    writes = []
    t0 = time.time()
    n_inst = 0
    try:
        fut = decode_pool.submit(_decode, batches[0], rgb_vis, need_depth) if batches else None
        for b, batch in enumerate(batches):
            t_rgb, t_depth = fut.result()
            if b + 1 < len(batches):   # batch b + 1 decodes while batch b renders and composites
                fut = decode_pool.submit(_decode, batches[b + 1], rgb_vis, need_depth)
            ppi = [im[6] for im in batch]
            n_inst += sum(len(p) for p in ppi)
            H, W = (int(s) for s in (t_rgb if rgb_vis else t_depth).shape[1:3])
            if meshes is None:   # no instance in the whole selection: the image itself, blended with nothing
                m_rgb = m_depth = None
                inst_off = np.zeros(len(batch) + 1, np.int64)
                dev = torch.device(device)
            else:
                dev = meshes.device
            with torch.cuda.device(dev):
                if meshes is not None:
                    m_rgb, m_depth, inst_off = render_instances(meshes, ppi, np.stack([im[2] for im in batch]), H, W,
                                                                obj_colors)
                d_rgb = t_rgb.to(dev, non_blocking=True) if rgb_vis else None
                d_depth = t_depth.to(dev, non_blocking=True) if need_depth else None
                res = composite_device(m_rgb, m_depth, inst_off, d_rgb, d_depth if need_depth else None, flags)
                host = {k: v.cpu().numpy() for k, v in res.items() if v is not None}
            outs = finish_host(host, inst_off, [[p.get("text_info") for p in ps] for ps in ppi], flags)
            for im, o in zip(batch, outs):
                d = os.path.join(vis_path, dataset, split, "{:06d}".format(im[0]))
                os.makedirs(d, exist_ok=True)
                if "rgb" in o:
                    writes.append(write_pool.submit(_save_jpg, os.path.join(d, "{:06d}.jpg".format(im[1])), o["rgb"]))
                if "depth_diff" in o:
                    writes.append(write_pool.submit(_save_jpg, os.path.join(d, "{:06d}_depth_diff.jpg".format(im[1])),
                                                    o["depth_diff"]))
        for f in writes:
            f.result()
    finally:
        decode_pool.shutdown(wait=True, cancel_futures=True)
        write_pool.shutdown(wait=True)
    return {"images": len(images), "instances": n_inst, "seconds": time.time() - t0}


def _ids(s):
    return None if s is None else [int(v) for v in s.split(",") if v]


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Visualise the GT poses (or a results CSV's estimates) of a BOP split on "
                                             "the GPU (vis_gt_poses.py without GL)")
    ap.add_argument("--dataset", default="lm")
    ap.add_argument("--dataset_split", default="test")
    ap.add_argument("--dataset_split_type", default=None)
    ap.add_argument("--targets_filename", default=None, help="targets JSON in the dataset folder (default: all images)")
    ap.add_argument("--scene_ids", default=None, help="comma-separated (default: every scene)")
    ap.add_argument("--im_ids", default=None, help="comma-separated (default: every image)")
    ap.add_argument("--gt_ids", default=None, help="comma-separated (default: every GT instance)")
    ap.add_argument("--no_vis_rgb", action="store_true")
    ap.add_argument("--no_resolve_visib", action="store_true")
    ap.add_argument("--no_depth_diff", action="store_true")
    ap.add_argument("--vis_orig_color", action="store_true", help="render the models' textures or vertex colours (grey without)")
    ap.add_argument("--shading", default="flat", help="flat (the only shading vis_gt_poses.py uses)")
    ap.add_argument("--colors_json", default=None, help="colour list, e.g. the BOP toolkit's colors.json")
    ap.add_argument("--result_filename", default=None, help="BOP results CSV: draw its estimates instead of GT")
    ap.add_argument("--vis_path", default=os.path.join("output", "vis_gt_poses"))
    ap.add_argument("--datasets_path", default=os.environ.get("BOP_PATH", "datasets/BOP_DATASETS/"))
    ap.add_argument("--models_dir", default=None, help="directory of obj_XXXXXX.ply (default: the split's models_eval)")
    ap.add_argument("--max_bytes", default=DEFAULT_MAX_BYTES, type=int, help="device memory budget of one batch")
    ap.add_argument("--renderer_type", default="cuda", help="accepted for compatibility; renders use the CUDA rasteriser")
    args = ap.parse_args(argv)
    if args.shading != "flat":
        ap.error("--shading {}: only flat shading is supported (phong has no caller in vis_gt_poses.py)".format(
            args.shading))
    args.scene_ids, args.im_ids, args.gt_ids = _ids(args.scene_ids), _ids(args.im_ids), _ids(args.gt_ids)
    if args.no_vis_rgb and args.no_depth_diff:
        ap.error("--no_vis_rgb and --no_depth_diff leave nothing to visualise")
    return args


def main(argv=None):
    args = parse_args(argv)
    sp = gt_info.split_params(args.datasets_path, args.dataset, args.dataset_split, args.dataset_split_type)
    targets = None
    if args.targets_filename is not None:
        with open(os.path.join(sp["base_path"], args.targets_filename)) as f:
            targets = {}
            for t in json.load(f):
                targets.setdefault(int(t["scene_id"]), set()).add(int(t["im_id"]))
    results, vis_path = None, args.vis_path
    if args.result_filename is not None:
        results = {}
        for r in bop_eval.load_bop_results(args.result_filename):
            results.setdefault((int(r["scene_id"]), int(r["im_id"])), []).append(
                {"obj_id": int(r["obj_id"]), "R": r["R"], "t": r["t"], "score": float(r["score"])})
        vis_path = os.path.join(vis_path, os.path.splitext(os.path.basename(args.result_filename))[0])
    colors = None
    if args.colors_json is not None:
        with open(args.colors_json) as f:
            colors = json.load(f)
    r = run_split(sp, gt_info.models_path(args.datasets_path, args.dataset, args.models_dir, "eval"), vis_path,
                  args.dataset, args.dataset_split, args.scene_ids, args.im_ids, args.gt_ids, targets, results,
                  not args.no_vis_rgb, not args.no_resolve_visib, not args.no_depth_diff, colors, args.vis_orig_color,
                  args.max_bytes)
    print(json.dumps({"split_path": sp["split_path"], **r, "images_per_s": r["images"] / max(r["seconds"], 1e-9)}))
    return r


if __name__ == "__main__":
    main()
