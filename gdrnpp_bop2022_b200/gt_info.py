"""Ground-truth annotations of a BOP split as batched GPU passes: scene_gt_info.json, mask/ and mask_visib/.

Mirrors the two BOP-toolkit scripts of the reference, without a GL context:
  * lib/pysixd/scripts/calc_gt_info.py   px_count_all / _valid / _visib, visib_fract, bbox_obj, bbox_visib per GT
                                          instance, from a render on a 3x canvas (principal point shifted by (W, H))
  * lib/pysixd/scripts/calc_gt_masks.py  mask/{im}_{gt}.png (dist_gt > 0) and mask_visib/{im}_{gt}.png (bop19)
Both renders come from the CUDA rasteriser (renderer.render_meshes, float z); one kernel (csrc/gt_info.cu) turns the
renders of many instances plus each image's sensor depth into integer counts, boxes and masks, with the distance and
bop19 visibility arithmetic VSD uses.  No CPU fallback: the GPU path needs CUDA and raises GdrnError otherwise.

  python -m gdrnpp_bop2022_b200.gt_info --dataset lmo --dataset_split train --dataset_split_type pbr
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
from ._lib import GdrnError

DEFAULT_MAX_BYTES = 2 << 30


def calc_2d_bbox(xs, ys):
    """The 2D box calc_gt_info.py stores, [x_min, y_min, x_max - x_min, y_max - y_min], unclipped and with no +1.

    The reference calls misc.calc_2d_bbox(xs, ys, im_size) but lib/pysixd/misc.py does not define it; this is the BOP
    toolkit's definition, which the script was forked from and which the shipped BOP scene_gt_info.json files follow.
    (The reference's own misc.calc_2d_bbox_xywh adds 1 to width and height; that is not what the BOP files hold.)"""
    x0, y0 = int(np.min(xs)), int(np.min(ys))
    return [x0, y0, int(np.max(xs)) - x0, int(np.max(ys)) - y0]


def _dist_im(depth, K):
    """misc.depth_im_to_dist_im_fast with Precomputer's pre_Xs / pre_Ys (f64)."""
    xs, ys = np.meshgrid(np.arange(depth.shape[1]), np.arange(depth.shape[0]))
    pre_x = (xs - K[0, 2]) / np.float64(K[0, 0])
    pre_y = (ys - K[1, 2]) / np.float64(K[1, 1])
    return np.sqrt(np.multiply(pre_x, depth) ** 2 + np.multiply(pre_y, depth) ** 2 + depth.astype(np.float64) ** 2)


def _visib_bop19(d_test, d_model, delta):
    """visibility.estimate_visib_mask_gt, bop19 mode."""
    d_diff = d_model.astype(np.float32) - d_test.astype(np.float32)
    return np.logical_and(np.logical_or(d_diff <= delta, d_test == 0), d_model > 0)


def host_annotation(depth_large, depth_img, depth_test, K, delta):
    """The scripts' per-instance math in numpy, for one instance: the reference the GPU kernel is tested against and the
    host arm of bench_gt_info.py (the product path never calls it).  depth_large [3H,3W] f32 render on the 3x canvas,
    depth_img [H,W] f32 image-size render (or None), depth_test [H,W] f32 sensor depth in mm, K [3,3].
    -> (info dict as scene_gt_info.json holds it, mask u8 0/255 or None, mask_visib u8 0/255 or None)."""
    H, W = depth_test.shape
    depth_gt = depth_large[H:2 * H, W:2 * W]
    dist_gt = _dist_im(depth_gt, K)
    dist_im = _dist_im(depth_test, K)
    visib_gt = _visib_bop19(dist_im, dist_gt, delta)
    obj_mask_gt_large = depth_large > 0
    px_count_all = int(np.sum(obj_mask_gt_large))
    px_count_valid = int(np.sum(dist_im[dist_gt > 0] > 0))
    px_count_visib = int(visib_gt.sum())
    visib_fract = px_count_visib / float(px_count_all) if px_count_all > 0 else 0.0
    bbox, bbox_visib = [-1, -1, -1, -1], [-1, -1, -1, -1]
    if px_count_visib > 0:
        ys, xs = obj_mask_gt_large.nonzero()
        bbox = calc_2d_bbox(xs - W, ys - H)
        ys, xs = visib_gt.nonzero()
        bbox_visib = calc_2d_bbox(xs, ys)
    info = {"px_count_all": px_count_all, "px_count_valid": px_count_valid, "px_count_visib": px_count_visib,
            "visib_fract": float(visib_fract), "bbox_obj": bbox, "bbox_visib": bbox_visib}
    if depth_img is None:
        return info, None, None
    dist_g2 = _dist_im(depth_img, K)
    return (info, 255 * (dist_g2 > 0).astype(np.uint8),
            255 * _visib_bop19(dist_im, dist_g2, delta).astype(np.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# In-memory API
def instance_bytes(H, W, info=True, masks=True):
    """Device bytes one instance takes in a pass: the float-z render and the rasteriser's 64-bit z-buffer for each
    canvas, the masks, and the counters."""
    b = 56
    if info:
        b += 9 * H * W * 12
    if masks:
        b += H * W * 14
    return b


def _depth_u16(depth, dev):
    """Sensor depth [N,H,W] as the kernel reads it: 16-bit unsigned (numpy uint16 or torch uint16 / int16 holding the
    same bits), on dev."""
    if torch.is_tensor(depth):
        if depth.dtype == torch.uint16:
            depth = depth.view(torch.int16)
        if depth.dtype != torch.int16:
            raise GdrnError(f"gt_info: sensor depth must be 16-bit unsigned, got {depth.dtype}")
        t = depth
    else:
        a = np.asarray(depth)
        if a.dtype != np.uint16:
            raise GdrnError(f"gt_info: sensor depth must be 16-bit unsigned, got {a.dtype}")
        t = torch.from_numpy(np.ascontiguousarray(a).view(np.int16))
    if t.ndim != 3:
        raise GdrnError(f"gt_info: sensor depth must be [N,H,W], got shape {tuple(t.shape)}")
    return t.to(dev, non_blocking=True).contiguous()


def annotate_device(meshes, obj_ids, R, t, inst_img, K, depth, depth_scale, delta=15.0, info=True, masks=False,
                    max_bytes=DEFAULT_MAX_BYTES, out=None):
    """Launch the annotation of n instances; no synchronisation.  meshes: bop_eval.VsdMeshes (obj_id -> mesh, mm);
    obj_ids [n], R [n,3,3], t [n,3] (mm), inst_img [n] (image of each instance); K [N,3,3], depth [N,H,W] u16 (host or
    CUDA), depth_scale [N].  Instances go through the renders in chunks of at most max_bytes (instance_bytes each),
    which changes no output.  out: optional u8 CUDA buffer of at least result_bytes(n, H, W, masks) bytes.
    -> (buffer, {counts [n,3] i64, boxes [n,8] i32, mask / mask_visib [n,H,W] u8 when masks}) as views of buffer."""
    from . import renderer

    if not (info or masks):
        raise GdrnError("gt_info: nothing to compute (info and masks both off)")
    dev = meshes.device
    n = len(obj_ids)
    with torch.cuda.device(dev):
        d_test = _depth_u16(depth, dev)
        N, H, W = (int(s) for s in d_test.shape)
        Ks = torch.as_tensor(np.asarray(K, np.float64).reshape(N, 3, 3)).to(dev).contiguous()
        scale = torch.as_tensor(np.asarray(depth_scale, np.float32).reshape(N)).to(dev)
        img = np.asarray(inst_img, np.int64).reshape(n)
        if n and (img.min() < 0 or img.max() >= N):
            raise GdrnError(f"gt_info: inst_img out of range [0, {N})")
        nbytes = result_bytes(n, H, W, masks)
        buf = out if out is not None else torch.empty(max(nbytes, 8), dtype=torch.uint8, device=dev)
        if buf.numel() < nbytes or not buf.is_cuda:
            raise GdrnError("gt_info: output buffer too small")
        res = _views(buf, n, H, W, masks)
        if n == 0:
            return buf, res
        try:
            ids = torch.tensor([meshes.ids[int(o)] for o in obj_ids], dtype=torch.int32, device=dev)
        except KeyError as e:
            raise GdrnError(f"gt_info: no mesh for obj_id {e.args[0]}") from None
        poses = torch.from_numpy(np.concatenate([np.asarray(R, np.float64).reshape(n, 3, 3),
                                                 np.asarray(t, np.float64).reshape(n, 3, 1)], axis=2)).to(dev)
        K_img = np.asarray(K, np.float64).reshape(N, 3, 3)[img]
        K_large = K_img.copy()
        K_large[:, 0, 2] += W
        K_large[:, 1, 2] += H
        K_img_t = torch.from_numpy(K_img).to(dev)
        K_large_t = torch.from_numpy(K_large).to(dev)
        img_t = torch.from_numpy(img.astype(np.int32)).to(dev)
        chunk = max(1, int(max_bytes) // instance_bytes(H, W, info, masks))
        L = _lib.lib()
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            d_large = renderer.render_meshes(ids[s:e], poses[s:e], K_large_t[s:e], 3 * H, 3 * W, bop_eval.VSD_ZNEAR,
                                             bop_eval.VSD_ZFAR, quantize_bits=0) if info else None
            d_img = renderer.render_meshes(ids[s:e], poses[s:e], K_img_t[s:e], H, W, bop_eval.VSD_ZNEAR,
                                           bop_eval.VSD_ZFAR, quantize_bits=0) if masks else None
            _lib.check(L.gdrn_gt_info(_lib.ptr(d_large), _lib.ptr(d_img), _lib.ptr(d_test), _lib.ptr(scale), _lib.ptr(Ks),
                                      _lib.ptr(img_t[s:e]), e - s, H, W, float(delta), _lib.ptr(res["counts"][s:e]),
                                      _lib.ptr(res["boxes"][s:e]),
                                      _lib.ptr(res["mask"][s:e]) if masks else None,
                                      _lib.ptr(res["mask_visib"][s:e]) if masks else None, _lib.current_stream()),
                       "gdrn_gt_info")
    return buf, res


def result_bytes(n, H, W, masks):
    """Bytes of one result buffer: counts [n,3] i64, boxes [n,8] i32, then the two masks [n,H,W] u8."""
    return n * 56 + (2 * n * H * W if masks else 0)


def _views(buf, n, H, W, masks):
    res = {"counts": buf[:n * 24].view(torch.int64).view(n, 3), "boxes": buf[n * 24:n * 56].view(torch.int32).view(n, 8)}
    if masks:
        HW = H * W
        res["mask"] = buf[n * 56:n * 56 + n * HW].view(n, H, W)
        res["mask_visib"] = buf[n * 56 + n * HW:n * 56 + 2 * n * HW].view(n, H, W)
    return res


def _host_result(res):
    """Counts and boxes of host views -> per-field numpy arrays with visib_fract formed in f64, as the script forms it."""
    counts = res["counts"].numpy()
    boxes = res["boxes"].numpy()
    out = {"px_count_all": counts[:, 0].copy(), "px_count_valid": counts[:, 1].copy(), "px_count_visib": counts[:, 2].copy(),
           "bbox_obj": boxes[:, :4].astype(np.int64), "bbox_visib": boxes[:, 4:].astype(np.int64)}
    with np.errstate(divide="ignore", invalid="ignore"):
        vf = out["px_count_visib"] / out["px_count_all"].astype(np.float64)
    out["visib_fract"] = np.where(out["px_count_all"] > 0, vf, 0.0)
    for k in ("mask", "mask_visib"):
        if k in res:
            out[k] = res[k].numpy()
    return out


def annotate(meshes, obj_ids, R, t, inst_img, K, depth, depth_scale, delta=15.0, masks=False, info=True,
             max_bytes=DEFAULT_MAX_BYTES):
    """GT annotations of n instances of N images in one batched call (see annotate_device for the arguments).
    -> {px_count_all, px_count_valid, px_count_visib [n] i64, visib_fract [n] f64, bbox_obj, bbox_visib [n,4] i64,
    and with masks: mask, mask_visib [n,H,W] u8 0 / 255}."""
    buf, _ = annotate_device(meshes, obj_ids, R, t, inst_img, K, depth, depth_scale, delta, info, masks, max_bytes)
    n = len(obj_ids)
    host = buf.cpu()
    H, W = (int(s) for s in tuple(depth.shape)[1:])
    return _host_result(_views(host, n, H, W, masks))


def info_records(res, i0, i1):
    """scene_gt_info.json entries of instances [i0, i1) of an annotate result."""
    return [{"px_count_all": int(res["px_count_all"][i]), "px_count_valid": int(res["px_count_valid"][i]),
             "px_count_visib": int(res["px_count_visib"][i]), "visib_fract": float(res["visib_fract"][i]),
             "bbox_obj": [int(v) for v in res["bbox_obj"][i]], "bbox_visib": [int(v) for v in res["bbox_visib"][i]]}
            for i in range(i0, i1)]


def save_json(path, content):
    """inout.save_json (sort=False): one top-level element per line; an empty dict is written as "{\\n}"."""
    if isinstance(content, dict) and not content:
        with open(path, "w") as f:
            f.write("{\n}")
        return
    bop_eval.save_json(path, content)


# ---------------------------------------------------------------------------------------------------------------------
# Split and model layout (dataset_params.get_split_params / get_model_params)
DATASETS = ("lm", "lmo", "tless", "tudl", "tyol", "ruapc", "icmi", "icbin", "itodd", "hbs", "hb", "ycbv", "ycbvposecnn",
            "hope")


def split_params(datasets_path, dataset, split, split_type=None):
    """-> {split_path, split_type, depth_ext} of one split, with get_split_params' defaults: T-LESS and HB take the
    primesense split type, TUD-L's train split render, YCB-V's train split real; ITODD depth images are .tif."""
    if dataset not in DATASETS:
        raise ValueError("Unknown BOP dataset ({}).".format(dataset))
    name = {"hbs": "hb", "ycbvposecnn": "ycbv"}.get(dataset, dataset)
    if split_type is None:
        if dataset in ("tless", "hb", "hbs"):
            split_type = "primesense"
        elif dataset == "tudl" and split == "train":
            split_type = "render"
        elif name == "ycbv" and split == "train":
            split_type = "real"
    split_path = os.path.join(datasets_path, name, split)
    if split_type is not None and split_type != "bb8":
        split_path += "_" + split_type
    depth_ext = ".tif" if dataset == "itodd" and split_type != "pbr" else ".png"
    # the colour image: rgb/ (JPEG for pbr), or for ITODD gray/ (.tif); vis_gt_poses.py reads rgb/ for any pbr split
    im_modality = "gray" if dataset == "itodd" and split_type != "pbr" else "rgb"
    im_ext = ".jpg" if split_type == "pbr" else (".tif" if im_modality == "gray" else ".png")
    return {"base_path": os.path.join(datasets_path, name), "split_path": split_path, "split_type": split_type,
            "depth_ext": depth_ext, "im_modality": im_modality, "im_ext": im_ext}


def models_path(datasets_path, dataset, models_dir=None, model_type=None):
    """The model directory the scripts render: models/ (models_cad/ for T-LESS), models_{model_type}/ when a model type
    is given (vis_gt_poses.py: "eval"), or models_dir when given."""
    if models_dir:
        return models_dir
    name = {"hbs": "hb", "ycbvposecnn": "ycbv"}.get(dataset, dataset)
    if model_type is None and dataset == "tless":
        model_type = "cad"
    return os.path.join(datasets_path, name, "models" + ("_" + model_type if model_type else ""))


def depth_path(split_path, scene_id, im_id, depth_ext):
    """calc_gt_info.py:96-101: the split's depth template, falling back from .tif to .png.  Raises when neither exists."""
    p = os.path.join(split_path, "{:06d}".format(scene_id), "depth", "{:06d}{}".format(im_id, depth_ext))
    if not os.path.exists(p):
        p2 = p.replace(".tif", ".png")
        if not os.path.exists(p2):
            raise GdrnError("missing depth image {}".format(p))
        p = p2
    return p


def image_path(sp, scene_id, im_id):
    """The colour (or ITODD gray) image of one view, as the split's rgb_tpath / gray_tpath names it.  Raises when it
    does not exist."""
    p = os.path.join(sp["split_path"], "{:06d}".format(scene_id), sp["im_modality"], "{:06d}{}".format(im_id, sp["im_ext"]))
    if not os.path.exists(p):
        raise GdrnError("missing {} image {}".format(sp["im_modality"], p))
    return p


def present_scene_ids(split_path):
    """dataset_params.get_present_scene_ids: every numbered directory of the split."""
    if not os.path.isdir(split_path):
        raise GdrnError("split directory {} does not exist".format(split_path))
    return sorted(int(d) for d in os.listdir(split_path) if d.isdigit() and os.path.isdir(os.path.join(split_path, d)))


def plan_split(sp, scene_ids=None, need_depth=True):
    """Every image of the selected scenes in order: [(scene_id, [image records])], image record = {im_id, depth path,
    K [3,3], depth_scale, gts}.  Rejects a missing depth image or depth_scale before any work.  need_depth=False (for
    tools that only render, such as gen_xyz) leaves depth and depth_scale out of the records and checks neither."""
    scenes = []
    for scene_id in (present_scene_ids(sp["split_path"]) if scene_ids is None else scene_ids):
        sdir = os.path.join(sp["split_path"], "{:06d}".format(scene_id))
        scene_gt = bop_eval.load_scene_gt(os.path.join(sdir, "scene_gt.json"))
        scene_cam = bop_eval.load_scene_camera(os.path.join(sdir, "scene_camera.json"))
        ims = []
        for im_id in sorted(scene_gt):
            cam = scene_cam.get(im_id)
            if cam is None:
                raise GdrnError("scene {} image {}: no entry in scene_camera.json".format(scene_id, im_id))
            rec = {"im_id": im_id, "K": cam["cam_K"], "gts": scene_gt[im_id]}
            if need_depth:
                if "depth_scale" not in cam:
                    raise GdrnError("scene {} image {}: scene_camera.json has no depth_scale".format(scene_id, im_id))
                rec["depth"] = depth_path(sp["split_path"], scene_id, im_id, sp["depth_ext"])
                rec["depth_scale"] = float(cam["depth_scale"])
            ims.append(rec)
        scenes.append((scene_id, ims))
    return scenes


def load_models(model_dir, obj_ids):
    """{obj_id: (verts, faces)} of the PLY models the instances use; rejects an obj_id without a model file."""
    from .ply import load_ply

    meshes = {}
    for o in sorted(obj_ids):
        p = os.path.join(model_dir, "obj_{:06d}.ply".format(o))
        if not os.path.exists(p):
            raise GdrnError("obj_id {}: no model file {}".format(o, p))
        m = load_ply(p)
        if "faces" not in m:
            raise GdrnError("obj_id {}: {} has no faces".format(o, p))
        meshes[o] = (m["pts"], m["faces"])
    return meshes


def read_depth(path):
    """A sensor depth image as stored (16-bit)."""
    import cv2

    d = cv2.imread(path, cv2.IMREAD_ANYDEPTH)
    if d is None:
        raise GdrnError("cannot read depth image {}".format(path))
    if d.dtype not in (np.uint16, np.uint8):
        raise GdrnError("depth image {} is {}, expected 16-bit unsigned".format(path, d.dtype))
    return d


# ---------------------------------------------------------------------------------------------------------------------
# Dataset driver: depth decode on a pool into pinned staging (batch k+1 while batch k runs), one H2D copy, the renders
# and the annotation kernel, one D2H copy, JSON / PNG writes on a pool overlapped with the next batch
def _batches(scenes, batch_images):
    """Whole images of one scene per batch: [(scene_id, [image records], last batch of the scene)]."""
    out = []
    for scene_id, ims in scenes:
        if not ims:
            out.append((scene_id, [], True))
        for k in range(0, len(ims), batch_images):
            out.append((scene_id, ims[k:k + batch_images], k + batch_images >= len(ims)))
    return out


class _Staging:
    """Two pinned host slots, grown on demand.  Pinned only where CUDA is present: host-side validation (a depth image
    of the wrong size) then still fails before any device work on a machine without one."""

    def __init__(self):
        self.slots = [None, None]

    def get(self, k, numel, dtype):
        s = self.slots[k]
        if s is None or s.numel() < numel or s.dtype != dtype:
            s = torch.empty(max(numel, 1), dtype=dtype, pin_memory=torch.cuda.is_available())
            self.slots[k] = s
        return s[:numel]


def _decode(batch, slot):
    scene_id, ims, _ = batch
    if not ims:
        return None
    first = read_depth(ims[0]["depth"])
    H, W = first.shape[:2]
    out = slot(len(ims) * H * W).view(len(ims), H, W)
    for k, im in enumerate(ims):
        d = first if k == 0 else read_depth(im["depth"])
        if d.shape != (H, W):
            raise GdrnError("depth image {} is {}x{}, other images of scene {} are {}x{}".format(
                im["depth"], d.shape[1], d.shape[0], scene_id, W, H))
        out[k].numpy()[...] = d.astype(np.uint16, copy=False).view(np.int16)
    return out


def _check_scene_size(sizes, scene_id, H, W, path):
    if sizes.setdefault(scene_id, (H, W)) != (H, W):
        h0, w0 = sizes[scene_id]
        raise GdrnError("depth image {} is {}x{}, other images of scene {} are {}x{}".format(path, W, H, scene_id, w0, h0))


def run_split(sp, model_dir, delta=15.0, what=("info", "masks"), scene_ids=None, max_bytes=DEFAULT_MAX_BYTES,
              batch_images=16, workers=8, device="cuda", log=None, meshes=None):
    """Annotate every GT instance of a split; writes scene_gt_info.json ("info") and mask/, mask_visib/ ("masks") in
    each scene directory.  meshes: a bop_eval.VsdMeshes of the split's models to reuse (default: loaded from model_dir).
    -> {"images": int, "instances": int, "seconds": float}."""
    import cv2

    do_info, do_masks = "info" in what, "masks" in what
    scenes = plan_split(sp, scene_ids)
    used = {int(g["obj_id"]) for _, ims in scenes for im in ims for g in im["gts"]}
    meshes_host = None if meshes is not None and used <= set(meshes.ids) else load_models(model_dir, used)
    batches = _batches(scenes, max(1, int(batch_images)))
    staging, outs = _Staging(), _Staging()
    decode_pool, write_pool = ThreadPoolExecutor(max(1, workers)), ThreadPoolExecutor(max(1, workers))
    infos, sizes, slot_writes = {}, {}, [[], []]
    t0 = time.time()
    n_images = n_inst = 0
    png = [cv2.IMWRITE_PNG_COMPRESSION, 3]

    def finish(p):
        nonlocal n_images, n_inst
        (scene_id, ims, last), host, ev, k, H, W = p
        if ev is not None:
            ev.synchronize()
        scene_info = infos.setdefault(scene_id, {})
        if ims:
            res = _host_result(_views(host, sum(len(im["gts"]) for im in ims), H, W, do_masks))
            sdir = os.path.join(sp["split_path"], "{:06d}".format(scene_id))
            i0 = 0
            for im in ims:
                i1 = i0 + len(im["gts"])
                if do_info:
                    scene_info[im["im_id"]] = info_records(res, i0, i1)
                if do_masks:
                    for g in range(i1 - i0):
                        for d, key in (("mask", "mask"), ("mask_visib", "mask_visib")):
                            path = os.path.join(sdir, d, "{:06d}_{:06d}.png".format(im["im_id"], g))
                            slot_writes[k].append(write_pool.submit(cv2.imwrite, path, res[key][i0 + g], png))
                i0 = i1
                n_images += 1
            n_inst += i0
        if last and do_info:
            path = os.path.join(sp["split_path"], "{:06d}".format(scene_id), "scene_gt_info.json")
            slot_writes[k].append(write_pool.submit(save_json, path, dict(sorted(scene_info.items()))))
            infos.pop(scene_id)

    try:
        for scene_id, _ in scenes:
            sdir = os.path.join(sp["split_path"], "{:06d}".format(scene_id))
            if do_masks:
                os.makedirs(os.path.join(sdir, "mask"), exist_ok=True)
                os.makedirs(os.path.join(sdir, "mask_visib"), exist_ok=True)
        fut = decode_pool.submit(_decode, batches[0], lambda n: staging.get(0, n, torch.int16)) if batches else None
        pending, h2d_done = None, [None, None]
        for b, batch in enumerate(batches):
            k = b % 2
            staged = fut.result()
            if b + 1 < len(batches):   # the next batch decodes into the other slot, once that slot's upload is done
                if h2d_done[1 - k] is not None:
                    h2d_done[1 - k].synchronize()
                fut = decode_pool.submit(_decode, batches[b + 1], lambda n, s=1 - k: staging.get(s, n, torch.int16))
            scene_id, ims, _ = batch
            if staged is None:
                if pending is not None:
                    finish(pending)
                pending = (batch, None, None, k, 0, 0)
                continue
            H, W = staged.shape[1:]
            _check_scene_size(sizes, scene_id, H, W, ims[0]["depth"])
            if meshes is None:
                meshes = bop_eval.VsdMeshes(meshes_host, device=device)
            dev = meshes.device
            with torch.cuda.device(dev):
                d_depth = staged.to(dev, non_blocking=True)   # the one H2D copy of the batch
                h2d_done[k] = torch.cuda.Event()
                h2d_done[k].record()
                gts = [(j, g) for j, im in enumerate(ims) for g in im["gts"]]
                n = len(gts)
                for f in slot_writes[k]:   # the host slot is reused: its earlier PNG / JSON writes must be done
                    f.result()
                slot_writes[k] = []
                buf = None
                if n:
                    buf, _ = annotate_device(
                        meshes, [int(g["obj_id"]) for _, g in gts],
                        np.stack([np.asarray(g["cam_R_m2c"], np.float64).reshape(3, 3) for _, g in gts]),
                        np.stack([np.asarray(g["cam_t_m2c"], np.float64).reshape(3) for _, g in gts]),
                        [j for j, _ in gts], np.stack([im["K"] for im in ims]), d_depth,
                        [im["depth_scale"] for im in ims], delta, do_info, do_masks, max_bytes)
                host = outs.get(k, result_bytes(n, H, W, do_masks), torch.uint8)
                ev = None
                if n:
                    host.copy_(buf[:host.numel()], non_blocking=True)   # the one D2H copy of the batch
                    ev = torch.cuda.Event()
                    ev.record()
            if pending is not None:
                finish(pending)
            pending = (batch, host, ev, k, H, W)
            if log:
                log("scene {} image {}: {} images, {} instances".format(scene_id, ims[-1]["im_id"], len(ims), n))
        if pending is not None:
            finish(pending)
        for fs in slot_writes:
            for f in fs:
                f.result()
    finally:
        decode_pool.shutdown(wait=True, cancel_futures=True)
        write_pool.shutdown(wait=True)
    return {"images": n_images, "instances": n_inst, "seconds": time.time() - t0}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Ground-truth annotations of a BOP split on the GPU "
                                             "(calc_gt_info.py and calc_gt_masks.py in one pass)")
    ap.add_argument("--dataset", default="lm")
    ap.add_argument("--dataset_split", default="test")
    ap.add_argument("--dataset_split_type", default=None)
    ap.add_argument("--datasets_path", default=os.environ.get("BOP_PATH", "datasets/BOP_DATASETS/"))
    ap.add_argument("--delta", default=15.0, type=float, help="tolerance of the visibility test [mm]")
    ap.add_argument("--what", default="info,masks", help="comma-separated: info (scene_gt_info.json), masks")
    ap.add_argument("--scene_ids", default=None, help="comma-separated scene ids (default: every scene of the split)")
    ap.add_argument("--models_dir", default=None, help="directory of obj_XXXXXX.ply (default: as the scripts pick)")
    ap.add_argument("--max_bytes", default=DEFAULT_MAX_BYTES, type=int, help="device memory budget of one render chunk")
    ap.add_argument("--batch_images", default=16, type=int, help="images per batch")
    ap.add_argument("--renderer_type", default="cuda", help="accepted for compatibility; renders always use the CUDA rasteriser")
    args = ap.parse_args(argv)
    args.what = [w for w in args.what.split(",") if w]
    bad = [w for w in args.what if w not in ("info", "masks")]
    if bad or not args.what:
        ap.error("--what takes info and / or masks, got {}".format(",".join(bad) or "nothing"))
    if args.scene_ids is not None:
        args.scene_ids = [int(s) for s in args.scene_ids.split(",") if s]
    return args


def main(argv=None):
    args = parse_args(argv)
    sp = split_params(args.datasets_path, args.dataset, args.dataset_split, args.dataset_split_type)
    r = run_split(sp, models_path(args.datasets_path, args.dataset, args.models_dir), args.delta, args.what,
                  args.scene_ids, args.max_bytes, args.batch_images)
    print(json.dumps({"split_path": sp["split_path"], **r, "images_per_s": r["images"] / max(r["seconds"], 1e-9)}))
    return r


if __name__ == "__main__":
    main()
