"""GT and estimated pose outlines over a BOP split's test images on the GPU: the per-dataset vis_poses_full scripts.

Mirrors core/gdrn_modeling/tools/ycbv/ycbv_3_vis_poses_full.py, tudl/tudl_vis_poses_full.py,
itodd/itodd_vis_poses_full.py and the zoomed ycbv/ycbv_2_vis_poses.py.  Per test image that has rows in the results CSV:
the estimates with score >= --score_thr are shaded into one image over the image's grey copy (EGLRenderer.render with
background=), every kept GT instance and every estimate is outlined alone (get_edge, bw = 3): estimate edges green,
else GT edges blue, else the shaded render.  {vis_dir}/{scene_id}_{im_id:06d}_vis0.png holds the image (zoomed with
--zoom, with the detection boxes of --det_file drawn), ..._vis1.png the composite.

Per batch of images of one size: one H2D copy, the zoom crops (native_ops.crop_resize_image), gdrn_vis_gray3, one
rast_render_scene_bg per image, one rast_render_meshes for every silhouette of the batch, gdrn_vis_outlines and one D2H
copy; only the detection boxes are drawn on the host, and the PNG writes run on a pool.

Decisions (the scripts differ from this where noted):
  * Estimates come from the BOP results CSV only.  GT instances are the ones the split's <ds>_bop_test registrar keeps:
    the images of test_targets_bop19.json (every image when the split has no targets file), instances whose
    mask_visib is not empty (scene_gt_info's px_count_visib > 0), and only images with at least one such instance.
    A split without scene_gt.json (ITODD, HB test) has no GT: every image is kept and only estimates are outlined.
  * GT rotations are cam_R_m2c in f32 (the scripts' quat2mat of the registrar's f32 quaternion is a ~1e-7 round trip
    that is not reproduced); GT t is f32(cam_t_m2c) / 1000 in f32, estimate t is t_mm / 1000 in f64, as the scripts.
  * The zoom box is the union of the kept GT instances' bbox_visib from scene_gt_info.json, taken to equal the
    mask2bbox_xyxy of their mask_visib PNGs (true of the files gt_info writes); no mask PNG is decoded.
  * Each image is rendered at its own size (the scripts hard-code 640 x 480 or 1280 x 960).
  * --det_file draws on the full-frame vis0 only; with --zoom it is refused (no script draws boxes on a zoomed image).

  python -m gdrnpp_bop2022_b200.vis_poses_full --dataset ycbv --result_filename gdrn_ycbv-test.csv
  python -m gdrnpp_bop2022_b200.vis_poses_full --dataset ycbv --result_filename gdrn_ycbv-test.csv --zoom
  python -m gdrnpp_bop2022_b200.vis_poses_full --dataset tudl --result_filename all_tudl-test.csv --det_file dets.json
"""
import argparse
import csv
import ctypes
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
from . import vis_poses
from ._lib import GdrnError

SCORE_THR = 0.3
OUT_SIZE = 512
EDGE_BW = 3
ZNEAR, ZFAR = 0.25, 6.0          # EGLRenderer's clip planes
CSV_COLUMNS = ("scene_id", "im_id", "obj_id", "score", "R", "t", "time")
BOX_BGR = (18, 127, 15)          # lib/vis_utils/image.py's _GREEN, vis_image_bboxes_cv2's box colour
TEXT_BGR = (0, 255, 0)           # mmcv.color_val("green"), its text colour


# ---------------------------------------------------------------------------------------------------------------------
# Host pieces: results CSV, zoom arithmetic, detection boxes
def load_results(path):
    """The results CSV as the scripts read it (pandas, by column name): {(scene_id, im_id): [{obj_id, score, R [3,3]
    f64, t [3] f64 in m}]} in file order.  Every row is kept; the score threshold applies when drawing."""
    with open(path, newline="") as f:
        rd = csv.DictReader(f)
        missing = [c for c in CSV_COLUMNS if c not in (rd.fieldnames or [])]
        if missing:
            raise GdrnError("results CSV {}: missing column(s) {}".format(path, ", ".join(missing)))
        out = {}
        for r in rd:
            out.setdefault((int(r["scene_id"]), int(r["im_id"])), []).append(
                {"obj_id": int(r["obj_id"]), "score": float(r["score"]),
                 "R": np.array([float(v) for v in r["R"].strip(" ").split(" ")]).reshape(3, 3),
                 "t": np.array([float(v) for v in r["t"].strip(" ").split(" ")]) / 1000})
    return out


def kept_estimates(rows, score_thr=SCORE_THR):
    """The rows the scripts draw: score >= score_thr, in file order."""
    return [r for r in rows if not r["score"] < score_thr]


def zoom_params(box_xyxy, K, imH, imW, out_size=OUT_SIZE):
    """ycbv_2_vis_poses.py:174-190 for the xyxy box (bottom-right pixel included) and the registrar's f32 K ->
    (center [2] f64, scale f64, M [2,3] f64 (crop_resize_by_warp_affine's forward map), K_zoom [3,3] f32)."""
    from .native_ops import get_affine_transform

    minx, miny, maxx, maxy = (np.int64(v) for v in box_xyxy)
    center = np.array([(minx + maxx) / 2, (miny + maxy) / 2])
    scale = max(maxx - minx, maxy - miny) * 1.5
    crop_minx = max(0, center[0] - scale / 2)
    crop_miny = max(0, center[1] - scale / 2)
    crop_maxx = min(imW - 1, center[0] + scale / 2)
    crop_maxy = min(imH - 1, center[1] + scale / 2)
    scale = min(scale, min(crop_maxx - crop_minx, crop_maxy - crop_miny))
    if not scale > 0:   # the scripts' warp would be singular
        raise GdrnError("--zoom: the zoom box {} is one pixel".format(tuple(int(v) for v in box_xyxy)))
    M = get_affine_transform(center, (scale, scale), 0, (out_size, out_size))   # crop_resize_by_warp_affine's tuple
    K_zoom = np.asarray(K, np.float32).copy()
    K_zoom[0, 2] -= center[0] - scale / 2
    K_zoom[1, 2] -= center[1] - scale / 2
    K_zoom[0, :] *= out_size / scale
    K_zoom[1, :] *= out_size / scale
    return center, scale, M, K_zoom


def det_boxes(dets, score_thr=SCORE_THR):
    """The tudl / itodd scripts' boxes from one image's detections (convert_det_to_our_format layout): score >=
    score_thr, bbox_est xywh -> xyxy, label str(obj_id)."""
    boxes, labels = [], []
    for d in dets:
        if d["score"] < score_thr:
            continue
        x1, y1, w1, h1 = d["bbox_est"]
        boxes.append(np.array([x1, y1, x1 + w1, y1 + h1]))
        labels.append(str(d["obj_id"]))
    return boxes, labels


def draw_bboxes(img, bboxes, labels=None, font_scale=0.5, font_thickness=2, box_thickness=2):
    """lib/vis_utils/image.py:vis_image_bboxes_cv2 with its defaults on a BGR u8 image: xyxy boxes (truncated to int32)
    in _GREEN, thickness 2, and each label in green at (x1, y1 - 2) -> a new u8 image."""
    import cv2

    out = img.copy()
    for i, bbox in enumerate(np.array(bboxes)):
        x1, y1, x2, y2 = (int(v) for v in bbox.astype(np.int32)[:4])
        cv2.rectangle(out, (x1, y1), (x2, y2), BOX_BGR, thickness=box_thickness)
        if labels is not None:
            cv2.putText(out, labels[i], (x1, y1 - 2), cv2.FONT_HERSHEY_SIMPLEX, font_scale, TEXT_BGR, font_thickness)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Split planning
def plan(sp, scene_ids=None, results=None, zoom=False, score_thr=SCORE_THR):
    """The images the scripts visit, in the registrar's order, that have rows in `results`:
    [(scene_id, im_id, K f32 [3,3], None, None, image path, instances, gt box xyxy or None)], instances = kept GT
    [{obj_id, R, t, gt: True}] then the drawn estimates [{..., gt: False}] (R, t in m).  See the module's decisions."""
    targets = None
    tpath = os.path.join(sp["base_path"], "test_targets_bop19.json")
    if os.path.exists(tpath):
        targets = {}
        for t in bop_eval.load_json(tpath):
            targets.setdefault(int(t["scene_id"]), set()).add(int(t["im_id"]))
    scenes = gt_info.present_scene_ids(sp["split_path"]) if scene_ids is None else scene_ids
    has_gt = all(os.path.exists(os.path.join(sp["split_path"], "{:06d}".format(s), "scene_gt.json")) for s in scenes)
    if zoom and not has_gt:
        raise GdrnError("--zoom: split {} has no GT (scene_gt.json), so no zoom box".format(sp["split_path"]))
    out = []
    if has_gt:
        infos = {}
        for im in vis_poses.plan_images(sp, scenes, targets=targets):
            scene_id, im_id = im[0], im[1]
            if scene_id not in infos:
                infos[scene_id] = bop_eval.load_json(os.path.join(sp["split_path"], "{:06d}".format(scene_id),
                                                                  "scene_gt_info.json"), keys_to_int=True)
            info = infos[scene_id].get(im_id)
            if info is None or len(info) != len(im[6]):
                raise GdrnError("scene {} image {}: scene_gt_info.json does not match scene_gt.json".format(scene_id,
                                                                                                           im_id))
            keep = [k for k in range(len(im[6])) if int(info[k]["px_count_visib"]) > 0]
            if not keep:   # the registrar drops an image without a kept instance
                continue
            gts = [{"obj_id": int(im[6][k]["obj_id"]), "gt": True,
                    "R": np.asarray(im[6][k]["R"], np.float32).reshape(3, 3),
                    "t": np.asarray(im[6][k]["t"], np.float32).reshape(3) / 1000.0} for k in keep]
            bb = np.array([info[k]["bbox_visib"] for k in keep], np.int64)
            box = (int(bb[:, 0].min()), int(bb[:, 1].min()), int((bb[:, 0] + bb[:, 2]).max()),
                   int((bb[:, 1] + bb[:, 3]).max()))
            out.append([scene_id, im_id, np.asarray(im[2], np.float32), im[5], gts, box])
    else:
        for scene_id in scenes:
            cams = bop_eval.load_scene_camera(os.path.join(sp["split_path"], "{:06d}".format(scene_id),
                                                           "scene_camera.json"))
            for im_id in sorted(cams):
                if targets is not None and im_id not in targets.get(scene_id, set()):
                    continue
                out.append([scene_id, im_id, np.asarray(cams[im_id]["cam_K"], np.float32), None, [], None])
    images = []
    for scene_id, im_id, K, path, gts, box in out:
        rows = results.get((scene_id, im_id)) if results is not None else []
        if results is not None and not rows:   # the scripts: "<scene>/<im> not detected", nothing written
            continue
        if zoom and box is None:
            raise GdrnError("--zoom: scene {} image {} has no kept GT instance".format(scene_id, im_id))
        if path is None:
            path = gt_info.image_path(sp, scene_id, im_id)
        ests = [{"obj_id": r["obj_id"], "gt": False, "R": r["R"], "t": r["t"]} for r in kept_estimates(rows or [], score_thr)]
        images.append((scene_id, im_id, K, None, None, path, gts + ests, box))
    return images


# ---------------------------------------------------------------------------------------------------------------------
# Device passes
def gray3(img, rgb_order=True, out=None):
    """gdrn_vis_gray3: [N,H,W,3] u8 CUDA (RGB, or BGR with rgb_order=False) -> the grey image stacked three times."""
    N, H, W = (int(s) for s in img.shape[:3])
    out = torch.empty_like(img) if out is None else out
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().gdrn_vis_gray3(_lib.ptr(img), N, H, W, int(bool(rgb_order)), _lib.ptr(out),
                                             _lib.current_stream()), "gdrn_vis_gray3")
    return out


def outlines(shaded, cover, inst_off, is_gt, bw=EDGE_BW, out=None):
    """gdrn_vis_outlines: shaded [N,H,W,3] f32 (render_scene "image", RGB in [0,1]), cover [n,H,W] f32 (or None when
    n = 0), inst_off [N+1] i32 and is_gt [n] u8 CUDA -> out [N,H,W,3] u8 BGR (see include/gdrn_b200.h)."""
    N, H, W = (int(s) for s in shaded.shape[:3])
    n = 0 if cover is None else int(cover.shape[0])
    out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=shaded.device) if out is None else out
    with torch.cuda.device(shaded.device):
        _lib.check(_lib.lib().gdrn_vis_outlines(_lib.ptr(shaded), _lib.ptr(cover), _lib.ptr(inst_off),
                                                _lib.ptr(is_gt), N, n, H, W, int(bw), _lib.ptr(out),
                                                _lib.current_stream()), "gdrn_vis_outlines")
    return out


def render_batch(models, batch, bg, Ks, H, W, out):
    """Device work of one batch after the background: per image one rast_render_scene_bg of its estimates over bg[j],
    one rast_render_meshes of every instance, then gdrn_vis_outlines into out [N,H,W,3] u8.  models: {obj_id: Model3D};
    Ks [N,3,3] f32 (host)."""
    from .renderer import EGL_MAT_AMBIENT, EGL_MAT_DIFFUSE

    dev, L = bg.device, _lib.lib()
    N = len(batch)
    insts = [(j, p) for j, im in enumerate(batch) for p in im[6]]
    n = len(insts)
    ids_h = np.array([models[p["obj_id"]].mesh_id for _, p in insts], np.int32)
    poses_h = np.zeros((n, 3, 4), np.float32)
    for k, (_, p) in enumerate(insts):
        poses_h[k, :, :3] = p["R"]
        poses_h[k, :, 3] = p["t"]
    inst_off_h = np.cumsum([0] + [len(im[6]) for im in batch]).astype(np.int32)
    is_gt_h = np.array([p["gt"] for _, p in insts], np.uint8)
    # one upload of the batch's small tables: ids, poses, K per instance, K per image, inst_off, is_gt
    meta = torch.from_numpy(np.concatenate([ids_h.view(np.uint8), poses_h.view(np.uint8).ravel(),
                                            Ks[[j for j, _ in insts]].astype(np.float32).view(np.uint8).ravel(),
                                            Ks.astype(np.float32).view(np.uint8).ravel(), inst_off_h.view(np.uint8),
                                            is_gt_h])).to(dev, non_blocking=False)
    o = 0

    def take(nbytes, dt):
        nonlocal o
        t = meta[o:o + nbytes].view(dt)
        o += nbytes
        return t

    ids, poses, Ki, Kim = take(4 * n, torch.int32), take(48 * n, torch.float32), take(36 * n, torch.float32), \
        take(36 * N, torch.float32)
    inst_off, is_gt = take(4 * (N + 1), torch.int32), take(n, torch.uint8)
    max_inst = max([len(im[6]) for im in batch] + [1])
    shaded = torch.empty((N, H, W, 3), dtype=torch.float32, device=dev)
    depth = torch.empty((H, W), dtype=torch.float32, device=dev)
    scratch = torch.empty((L.rast_scene_scratch_bytes(max_inst, H, W) + 7) // 8, dtype=torch.int64, device=dev)
    light = (ctypes.c_float * 12)(0.0, 0.0, 0.0, 1.0, 1.0, 1.0, *EGL_MAT_DIFFUSE, *EGL_MAT_AMBIENT)
    stream = _lib.current_stream()
    for j, im in enumerate(batch):
        k0, k1 = int(inst_off_h[j]), int(inst_off_h[j + 1])
        est = [k for k in range(k0, k1) if not is_gt_h[k]]
        e0 = est[0] if est else k0   # the estimates of an image are contiguous, after its GT instances
        _lib.check(L.rast_render_scene_bg(_lib.ptr(ids[e0:]) if est else None,
                                          _lib.ptr(poses[12 * e0:]) if est else None, len(est),
                                          _lib.ptr(Kim[9 * j:]), H, W, ZNEAR, ZFAR, light, _lib.ptr(bg[j]),
                                          _lib.ptr(depth), None, None, None, _lib.ptr(shaded[j]), None,
                                          _lib.ptr(scratch), stream), "rast_render_scene_bg")
    cover = None
    if n:
        cover = torch.empty((n, H, W), dtype=torch.float32, device=dev)
        zb = torch.empty((n * H * W,), dtype=torch.int64, device=dev)
        _lib.check(L.rast_render_meshes(_lib.ptr(ids), _lib.ptr(poses), _lib.ptr(Ki), n, H, W, ZNEAR, ZFAR, 0,
                                        _lib.ptr(cover), None, _lib.ptr(zb), stream), "rast_render_meshes")
    return outlines(shaded, cover, inst_off, is_gt, EDGE_BW, out)


# ---------------------------------------------------------------------------------------------------------------------
# Driver
def _write_png(path, bgr):
    import cv2

    if not cv2.imwrite(path, np.ascontiguousarray(bgr)):
        raise GdrnError("cannot write {}".format(path))


def load_models(model_dir, obj_ids, device):
    """{obj_id: Model3D} shaded as EGLRenderer loads them (vertex_scale 0.001), with obj_{id:06d}.png beside a model as
    its texture when that file exists (the ycbv scripts pass those; the others pass none)."""
    from .renderer import load_models as _load

    paths, tex = [], []
    for o in sorted(obj_ids):
        p = os.path.join(model_dir, "obj_{:06d}.ply".format(o))
        if not os.path.exists(p):
            raise GdrnError("obj_id {}: no model file {}".format(o, p))
        t = os.path.join(model_dir, "obj_{:06d}.png".format(o))
        paths.append(p)
        tex.append(t if os.path.exists(t) else "")
    return dict(zip(sorted(obj_ids), _load(paths, scale_to_meter=0.001, device=device, texture_paths=tex,
                                           shading=True)))


def run_split(sp, model_dir, vis_dir, results, zoom=False, out_size=OUT_SIZE, dets=None, score_thr=SCORE_THR,
              scene_ids=None, max_bytes=vis_poses.DEFAULT_MAX_BYTES, workers=8, device="cuda", models=None):
    """Write {vis_dir}/{scene_id}_{im_id:06d}_vis0.png / _vis1.png for every image of the split with rows in `results`
    (load_results).  dets: {"scene/im": [{bbox_est, obj_id, score}]} boxes drawn on vis0.  -> {images, instances,
    seconds}."""
    from .native_ops import crop_resize_image

    if zoom and dets is not None:
        raise GdrnError("--det_file with --zoom: the boxes are drawn on the full-frame image only")
    images = plan(sp, scene_ids, results, zoom, score_thr)
    used = sorted({p["obj_id"] for im in images for p in im[6]})
    dev = torch.device(device)
    if models is None:
        models = load_models(model_dir, used, dev)
    missing = [o for o in used if o not in models]
    if missing:
        raise GdrnError("obj_id {}: no model".format(missing[0]))
    os.makedirs(vis_dir, exist_ok=True)
    batches = vis_poses._batches(images, max_bytes, False)
    decode_pool, write_pool = ThreadPoolExecutor(max(1, workers)), ThreadPoolExecutor(max(1, workers))
    writes, n_inst, t0 = [], 0, time.time()
    try:
        fut = decode_pool.submit(vis_poses._decode, batches[0], True, False) if batches else None
        for b, batch in enumerate(batches):
            t_rgb, _ = fut.result()
            if b + 1 < len(batches):   # batch b + 1 decodes while batch b runs
                fut = decode_pool.submit(vis_poses._decode, batches[b + 1], True, False)
            N, H0, W0 = (int(s) for s in t_rgb.shape[:3])
            n_inst += sum(len(im[6]) for im in batch)
            with torch.cuda.device(dev):
                d_rgb = t_rgb.to(dev, non_blocking=True)
                H, W = (out_size, out_size) if zoom else (H0, W0)
                res = torch.empty((2 if zoom else 1, N, H, W, 3), dtype=torch.uint8, device=dev)
                if zoom:
                    Ks = []
                    for j, im in enumerate(batch):
                        _, _, M, Kz = zoom_params(im[7], im[2], H0, W0, out_size)
                        z = crop_resize_image(d_rgb[j], M[None], out_size, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
                        res[1, j] = z[0].permute(1, 2, 0).to(torch.uint8)
                        Ks.append(Kz)
                    img, Ks = res[1], np.stack(Ks)
                else:
                    img, Ks = d_rgb, np.stack([im[2] for im in batch])
                bg = gray3(img, rgb_order=True)
                render_batch(models, batch, bg, Ks, H, W, res[0])
                host = res.cpu().numpy()
            for j, im in enumerate(batch):
                stem = os.path.join(vis_dir, "{}_{:06d}".format(im[0], im[1]))
                vis0 = (host[1, j] if zoom else t_rgb[j].numpy())[..., ::-1]   # RGB -> BGR
                if dets is not None:   # an image missing from the file gets no box
                    vis0 = draw_bboxes(np.ascontiguousarray(vis0),
                                       *det_boxes(dets.get("{}/{}".format(im[0], im[1]), []), score_thr))
                writes.append(write_pool.submit(_write_png, stem + "_vis0.png", vis0))
                writes.append(write_pool.submit(_write_png, stem + "_vis1.png", host[0, j]))
        for f in writes:
            f.result()
    finally:
        decode_pool.shutdown(wait=True, cancel_futures=True)
        write_pool.shutdown(wait=True)
    return {"images": len(images), "instances": n_inst, "seconds": time.time() - t0}


def _ids(s):
    return None if s is None else [int(v) for v in s.split(",") if v]


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Draw GT and estimated pose outlines over a BOP test split's images on "
                                             "the GPU (the per-dataset vis_poses_full scripts)")
    ap.add_argument("--dataset", required=True, choices=gt_info.DATASETS)
    ap.add_argument("--result_filename", required=True, help="BOP results CSV (scene_id,im_id,obj_id,score,R,t,time)")
    ap.add_argument("--zoom", action="store_true", help="crop to the GT's visible box, as ycbv_2_vis_poses.py")
    ap.add_argument("--out_size", default=OUT_SIZE, type=int, help="side of the zoomed images")
    ap.add_argument("--det_file", default=None, help="detections {\"scene/im\": [{bbox_est, obj_id, score}]} to box on vis0")
    ap.add_argument("--score_thr", default=SCORE_THR, type=float)
    ap.add_argument("--vis_path", default=os.path.join("output", "vis_poses_full"))
    ap.add_argument("--datasets_path", default=os.environ.get("BOP_PATH", "datasets/BOP_DATASETS/"))
    ap.add_argument("--models_dir", default=None, help="directory of obj_XXXXXX.ply (default: the dataset's models/)")
    ap.add_argument("--scene_ids", default=None, help="comma-separated (default: every scene)")
    ap.add_argument("--max_bytes", default=vis_poses.DEFAULT_MAX_BYTES, type=int, help="device memory budget of one batch")
    args = ap.parse_args(argv)
    if args.out_size <= 0:
        ap.error("--out_size must be positive")
    if args.zoom and args.det_file is not None:
        ap.error("--det_file with --zoom: the boxes are drawn on the full-frame image only")
    args.scene_ids = _ids(args.scene_ids)
    return args


def main(argv=None):
    args = parse_args(argv)
    sp = gt_info.split_params(args.datasets_path, args.dataset, "test")
    if not os.path.exists(args.result_filename):
        raise GdrnError("results CSV {} does not exist".format(args.result_filename))
    results = load_results(args.result_filename)
    dets = None
    if args.det_file is not None:
        with open(args.det_file) as f:
            dets = json.load(f)
    vis_dir = os.path.join(args.vis_path, os.path.splitext(os.path.basename(args.result_filename))[0])
    r = run_split(sp, gt_info.models_path(args.datasets_path, args.dataset, args.models_dir), vis_dir, results,
                  args.zoom, args.out_size, dets, args.score_thr, args.scene_ids, args.max_bytes)
    print(json.dumps({"split_path": sp["split_path"], "vis_dir": vis_dir, **r,
                      "images_per_s": r["images"] / max(r["seconds"], 1e-9)}))
    return r


if __name__ == "__main__":
    main()
