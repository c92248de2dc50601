"""The dataset test loop of the reference (test_gdrn.sh -> main_gdrn.py --eval-only -> gdrn_inference_on_dataset ->
GDRN_Evaluator.process -> results CSV -> VAL.SCRIPT_PATH; engine/gdrn_evaluator.py:155-240, 668-810,
engine/test_utils.py:33-80), with the ROIs of many images in each forward.

  * images: the sorted unique (scene_id, im_id) pairs of VAL.TARGETS_FILENAME (datasets/*_bop_test.py), cam_K and
    depth_scale from each scene's scene_camera.json;
  * detections: load_detections_into_dataset (core/utils/dataset_utils.py:146-235);
  * batches: whole images, at most ``max_batch`` ROIs each (an image with more goes alone and the forward chunks it),
    images of one size per batch.  Host decoding runs in a thread pool into pinned staging for batch k+1 while batch k
    runs; per batch: one H2D copy, gdrn_roi_setup + gdrn_roi_crop_multi (native_ops.roi_batch_inputs), the forward (a
    CUDA graph per batch size), the evaluator's post-processing dispatch, one D2H copy of the poses;
  * results: one row per ROI, image order then ROI order, written with bop_eval.write_bop_results_csv and scored
    in-process with eval_pose_results_more.run.

Deviation from the reference: the ``time`` column of an image is its detection time plus its share of its batch's wall
time (batch time / images in the batch), since the reference times one image per forward.
"""
import json
import os
import threading
import time
from collections.abc import Mapping
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import bop_eval
from .gdrn_model import _cfg_get
from .native_ops import roi_batch_buffers, roi_batch_inputs
from .per_object import PerObjectGDRN

# obj_ids in label order: the `objects` lists of the reference's ref/<dataset>.py (hb: ref/hb_bop19.py)
DATASET_OBJ_IDS = {
    "lmo": [1, 5, 6, 8, 9, 10, 11, 12],
    "hb": [1, 3, 4, 8, 9, 10, 12, 15, 17, 18, 19, 22, 23, 29, 32, 33],
    "ycbv": list(range(1, 22)),
    "tless": list(range(1, 31)),
    "tudl": [1, 2, 3],
    "icbin": [1, 2],
    "itodd": list(range(1, 29)),
}
# image split directory where it differs from VAL.SPLIT (+ _SPLIT_TYPE), and (colour dir, extension) per dataset
IMAGE_SPLIT_DIRS = {"tless": "test_primesense", "hb": "test_primesense"}
IMAGE_DIRS = {"itodd": ("gray", ".tif")}


def cfg_get(cfg, path, default=None):
    return _cfg_get(cfg, path, default)


# ------------------------------------------------------------------------------------------------ configuration
def _resize_shortest_edge_size(h, w, short, max_size):
    """detectron2 ResizeShortestEdge.get_output_shape."""
    scale = short * 1.0 / min(h, w)
    newh, neww = (short, scale * w) if h < w else (scale * h, short)
    if max(newh, neww) > max_size:
        scale = max_size * 1.0 / max(newh, neww)
        newh, neww = newh * scale, neww * scale
    return int(newh + 0.5), int(neww + 0.5)


def check_config(cfg, im_size=None):
    """Reject the settings this loop does not implement, naming the setting.  im_size (H, W): also require the
    test-time ResizeShortestEdge to be the identity for that size."""
    def bad(msg):
        raise NotImplementedError(msg)

    if str(cfg_get(cfg, "TEST.TEST_BBOX_TYPE", "est")) == "gt":
        bad('TEST.TEST_BBOX_TYPE="gt": the test loop runs on detections (TEST_BBOX_TYPE="est")')
    if cfg_get(cfg, "TEST.COLOR_AUG", False):
        bad("TEST.COLOR_AUG=True: test-time colour augmentation is not supported")
    if str(cfg_get(cfg, "MODEL.POSE_NET.PNP_NET.COORD_2D_TYPE", "abs")) == "rel":
        bad('MODEL.POSE_NET.PNP_NET.COORD_2D_TYPE="rel" is not supported (only "abs")')
    if "depth" in str(cfg_get(cfg, "MODEL.POSE_NET.NAME", "")).lower():
        bad(f"MODEL.POSE_NET.NAME={cfg_get(cfg, 'MODEL.POSE_NET.NAME')!r}: depth as a network input is not supported")
    if not cfg_get(cfg, "VAL.USE_BOP", False):
        bad("VAL.USE_BOP=False selects GDRN_EvaluatorCustom, which is not supported (set VAL.USE_BOP=True)")
    if cfg_get(cfg, "VAL.EVAL_CACHED", False):
        bad("VAL.EVAL_CACHED=True (re-evaluating cached predictions) is not supported")
    if im_size is not None and cfg_get(cfg, "INPUT.IMG_AUG_RESIZE", True):
        short, max_size = cfg_get(cfg, "INPUT.MIN_SIZE_TEST", 480), cfg_get(cfg, "INPUT.MAX_SIZE_TEST", 640)
        short = short[-1] if isinstance(short, (list, tuple)) else short
        if short and _resize_shortest_edge_size(im_size[0], im_size[1], short, max_size) != tuple(im_size):
            bad(f"INPUT.MIN_SIZE_TEST={short} / INPUT.MAX_SIZE_TEST={max_size} resize {im_size[1]}x{im_size[0]} images; "
                "only the identity resize is supported")


def exp_id(cfg, config_file):
    """main_gdrn.py:122-131."""
    e = os.path.splitext(os.path.basename(config_file))[0]
    if cfg_get(cfg, "TEST.USE_PNP", False):
        return e + "{}_test".format(str(cfg_get(cfg, "TEST.PNP_TYPE", "ransac_pnp")).upper())
    return e + "_test"


def result_csv_name(cfg, exp_id_str, name="iter0"):
    """save_and_eval_results (test_utils.py:33-50)."""
    split_type = cfg_get(cfg, "VAL.SPLIT_TYPE", "")
    split_type_str = f"-{split_type}" if split_type else ""
    return "{}-{}_{}-{}{}.csv".format(exp_id_str.replace("_", "-"), name, cfg_get(cfg, "VAL.DATASET_NAME"),
                                      cfg_get(cfg, "VAL.SPLIT", "test"), split_type_str)


def label_obj_ids(dataset, targets=None):
    """obj_id of every label: the dataset's object list, or the sorted ids of the targets for other datasets."""
    if dataset in DATASET_OBJ_IDS:
        return list(DATASET_OBJ_IDS[dataset])
    return sorted({int(t["obj_id"]) for t in targets})


def resolve_path(path, datasets_root):
    """Paths that start with ``datasets/`` are relative to the reference's datasets directory."""
    return os.path.join(datasets_root, path[len("datasets/"):]) if path.startswith("datasets/") else path


# ------------------------------------------------------------------------------------------------ images / detections
def image_list(targets):
    """Sorted unique (scene_id, im_id) pairs of a targets file (datasets/ycbv_bop_test.py:108-110)."""
    return sorted({(int(t["scene_id"]), int(t["im_id"])) for t in targets})


def load_detections(detections, images, obj_ids, score_thr=0.0, top_k_per_obj=1, train_obj_ids=None):
    """load_detections_into_dataset: detections {"scene/im": [{obj_id, bbox_est, score, time}, ...]} ->
    [(image index, [det, ...])] for the images present in the file (an empty list keeps the image without ROIs).
    A det is {label, obj_id, bbox_est (xywh), score, time}; per object, the top_k_per_obj by score (stable on ties),
    objects in label order."""
    out = []
    for idx, (scene_id, im_id) in enumerate(images):
        key = f"{scene_id}/{im_id}"
        if key not in detections:
            continue
        per_obj = {o: [] for o in obj_ids}
        for det in detections[key]:
            oid = int(det["obj_id"])
            score = det.get("score", 1.0)
            if score < score_thr:
                continue
            if oid not in per_obj:
                continue
            if train_obj_ids is not None and oid not in train_obj_ids:
                continue
            per_obj[oid].append({"label": obj_ids.index(oid), "obj_id": oid, "bbox_est": det["bbox_est"], "score": score,
                                 "time": det.get("time", 0.0)})
        anns = []
        for o in obj_ids:
            cur = per_obj[o]
            anns.extend([a for _, a in sorted(zip([a["score"] for a in cur], cur), key=lambda p: p[0], reverse=True)]
                        [:top_k_per_obj])
        out.append((idx, anns))
    return out


def pack_batches(counts, max_batch, keys=None):
    """Whole images into batches of at most max_batch ROIs; an image with more goes alone.  keys: one hashable per
    image (its size); a batch holds images of one key.  -> [[image position, ...], ...]"""
    batches, cur, n, cur_key = [], [], 0, None
    for i, c in enumerate(counts):
        k = keys[i] if keys is not None else None
        if cur and (n + c > max_batch or k != cur_key):
            batches.append(cur)
            cur, n = [], 0
        cur.append(i)
        n += c
        cur_key = k
    if cur:
        batches.append(cur)
    return batches


def read_image(path):
    """BGR uint8 as read_image_mmcv(path, "BGR") reads it; a single-channel 8-bit image stays [H,W,1] (the crop kernel
    replicates it to three channels)."""
    import cv2

    im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if im is None:
        raise FileNotFoundError(path)
    if im.dtype != np.uint8 or (im.ndim == 3 and im.shape[2] != 3):
        im = cv2.imread(path, cv2.IMREAD_COLOR)
    return im.reshape(im.shape[0], im.shape[1], -1)


def image_shape(path):
    """(H, W, C) read_image returns for a file, from its header: C = 1 for 8-bit single-channel images."""
    from PIL import Image

    with Image.open(path) as im:
        return im.size[1], im.size[0], 1 if im.mode == "L" else 3


def read_depth(path):
    import cv2

    d = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if d is None:
        raise FileNotFoundError(path)
    if d.dtype != np.uint16:
        raise ValueError(f"{path}: depth must be 16-bit, got {d.dtype}")
    return d


class TestSet:
    """Images, cameras and detections of one BOP test split, as the reference's *_bop_test.py + detection loader
    build them."""

    def __init__(self, cfg, datasets_root, train_obj_ids=None):
        self.dataset = cfg_get(cfg, "VAL.DATASET_NAME")
        split, split_type = cfg_get(cfg, "VAL.SPLIT", "test"), cfg_get(cfg, "VAL.SPLIT_TYPE", "")
        self.bop_root = os.path.join(datasets_root, "BOP_DATASETS")
        self.base = os.path.join(self.bop_root, self.dataset)
        self.split_dir = os.path.join(self.base, IMAGE_SPLIT_DIRS.get(self.dataset, split + (f"_{split_type}" if split_type else "")))
        targets = bop_eval.load_json(os.path.join(self.base, cfg_get(cfg, "VAL.TARGETS_FILENAME", "test_targets_bop19.json")))
        self.images = image_list(targets)
        self.obj_ids = label_obj_ids(self.dataset, targets)
        color_dir, ext = IMAGE_DIRS.get(self.dataset, ("rgb", ".png"))
        cams = {}
        self._extents = {}
        self.K, self.depth_factor, self.rgb, self.depth = [], [], [], []
        for scene_id, im_id in self.images:
            sdir = os.path.join(self.split_dir, f"{scene_id:06d}")
            if scene_id not in cams:
                cams[scene_id] = bop_eval.load_json(os.path.join(sdir, "scene_camera.json"))
            cam = cams[scene_id][str(im_id)]
            self.K.append(np.array(cam["cam_K"], np.float32).reshape(3, 3))
            self.depth_factor.append(1000.0 / cam.get("depth_scale", 1.0))
            self.rgb.append(os.path.join(sdir, color_dir, f"{im_id:06d}{ext}"))
            self.depth.append(os.path.join(sdir, "depth", f"{im_id:06d}{ext}"))
        det_files = cfg_get(cfg, "DATASETS.DET_FILES_TEST", ())
        if not det_files:
            raise ValueError("DATASETS.DET_FILES_TEST is empty: the test loop reads its detections from a file")
        with open(resolve_path(det_files[0], datasets_root)) as f:
            dets = json.load(f)
        self.records = load_detections(dets, self.images, self.obj_ids, cfg_get(cfg, "DATASETS.DET_THR", 0.0),
                                       cfg_get(cfg, "DATASETS.DET_TOPK_PER_OBJ", 1), train_obj_ids)

    def extents(self, device):
        """[nc,3] float32 extents per label in metres from models_info (the loader's _get_extents: size_x/y/z)."""
        key = str(device)
        if key not in self._extents:
            info = bop_eval.load_json(os.path.join(self.base, "models_eval", "models_info.json"), keys_to_int=True)
            self._extents[key] = torch.tensor([[info[o]["size_" + c] / 1000.0 for c in "xyz"] for o in self.obj_ids],
                                              dtype=torch.float32).to(device)
        return self._extents[key]

    def meshes(self, device):
        """Meshes of models_eval in metres, in label order (the evaluator's depth-refine models)."""
        return [_mesh(os.path.join(self.base, "models_eval"), oid, str(device)) for oid in self.obj_ids]


_MESHES = {}


def _mesh(models_path, obj_id, device):
    """One Model3D per (models_eval directory, object, device) for the life of the process, so that a test loop run
    again in the same process does not read and upload its models again."""
    from .ply import load_ply
    from .renderer import Model3D

    key = (models_path, obj_id, device)
    if key not in _MESHES:
        m = load_ply(os.path.join(models_path, "obj_{:06d}.ply".format(obj_id)))
        _MESHES[key] = Model3D(m["pts"].astype(np.float32) * np.float32(0.001), m["faces"], device=device)
    return _MESHES[key]


# ------------------------------------------------------------------------------------------------ the loop
class _Stage:
    """One pinned host block + one device block for a batch: images, depth, ROI metadata, cameras."""

    def __init__(self, device):
        self.device = device
        self.host = torch.empty(0, dtype=torch.uint8).pin_memory()
        self.dev = torch.empty(0, dtype=torch.uint8, device=device)
        self.h2d_done = None

    def layout(self, N, H, W, C, n, with_depth):
        parts = [("images", (N, H, W, C), torch.uint8), ("K", (N, 3, 3), torch.float32),
                 ("det_meta", (n, 2), torch.int32), ("bbox_est", (n, 4), torch.float32)]
        if with_depth:
            parts += [("depth", (N, H, W), torch.uint16), ("depth_factor", (N,), torch.float64)]
        offs, o = {}, 0
        for name, shape, dt in parts:
            nb = int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size()
            offs[name] = (o, nb, shape, dt)
            o += (nb + 255) // 256 * 256
        if self.host.numel() < o:
            self.host = torch.empty(o, dtype=torch.uint8).pin_memory()
            self.dev = torch.empty(o, dtype=torch.uint8, device=self.device)
        self.nbytes = o
        view = lambda buf: {k: buf[a:a + nb].view(dt).view(shape) for k, (a, nb, shape, dt) in offs.items()}
        self.h, self.d = view(self.host), view(self.dev)


def _forward(model, st, graphs, use_cuda_graph):
    kw = dict(roi_classes=st["roi_cls"], roi_cams=st["roi_cam"], roi_whs=st["roi_wh"], roi_centers=st["roi_center"],
              resize_ratios=st["resize_ratio"], roi_coord_2d=st["roi_coord_2d"], roi_extents=st["roi_extent"])
    n = st["roi_img"].shape[0]
    if isinstance(model, PerObjectGDRN) or not use_cuda_graph or n > model.max_batch:
        return model(st["roi_img"], **kw)
    g = graphs.get(n)
    if g is None:
        g = graphs[n] = model.capture_graph({"roi_img": st["roi_img"], "roi_classes": st["roi_cls"],
                                             "roi_coord_2d": st["roi_coord_2d"], "roi_cams": st["roi_cam"],
                                             "roi_centers": st["roi_center"], "roi_whs": st["roi_wh"],
                                             "roi_extents": st["roi_extent"], "resize_ratios": st["resize_ratio"]})
    replay, out = g
    replay()
    return out


def postprocess(cfg, inp, out, meshes=None, mask_thr=0.5):
    """GDRN_Evaluator.process's dispatch (gdrn_evaluator.py:155-180): TEST.USE_PNP -> the PNP_TYPE branch and nothing
    after it; else TEST.USE_DEPTH_REFINE -> depth refine; else the network pose.  -> (rot [n,3,3], trans [n,3])."""
    rot, trans = out["rot"], out["trans"]
    n = rot.shape[0]
    if n == 0:
        return rot, trans
    if cfg_get(cfg, "TEST.USE_PNP", False):
        from .pnp_ransac import PNP_NET_TYPES, pnp_net_from_maps, pnp_ransac_from_maps

        t = str(cfg_get(cfg, "TEST.PNP_TYPE", "ransac_pnp")).lower()
        maps = (out["coor_x"], out["coor_y"], out["coor_z"], out["mask"], inp["roi_coord_2d"], inp["im_H"], inp["im_W"],
                inp["roi_extent"], inp["roi_cam"])
        if t == "ransac_pnp":
            poses = pnp_ransac_from_maps(*maps, mask_thr=mask_thr)
        elif t in PNP_NET_TYPES:
            poses = pnp_net_from_maps(*maps, rot, trans, pnp_type=t, mask_thr=mask_thr)
        else:
            raise NotImplementedError(f"TEST.PNP_TYPE {t!r}")
        return poses[:, :, :3], poses[:, :, 3]
    if cfg_get(cfg, "TEST.USE_DEPTH_REFINE", False):
        from .renderer import depth_refine, get_K_crop_resize

        if meshes is None:
            raise RuntimeError("TEST.USE_DEPTH_REFINE needs the object meshes")
        crop_xy = inp["roi_center"] - inp["scale"].view(n, 1) / 2
        K_crop = get_K_crop_resize(inp["roi_cam"], crop_xy, (64.0 / inp["scale"]).view(n, 1))
        xyz = torch.cat([out["coor_x"], out["coor_y"], out["coor_z"]], dim=1)
        trans = depth_refine(meshes, rot, trans, K_crop, xyz, out["mask"], inp["depth_sensor"],
                             iters=cfg_get(cfg, "TEST.DEPTH_REFINE_ITER", 2),
                             thresh=cfg_get(cfg, "TEST.DEPTH_REFINE_THRESHOLD", 0.8), mesh_ids=inp["roi_cls"],
                             coor_z_refine=bool(cfg_get(cfg, "TEST.USE_COOR_Z_REFINE", False)))
    return rot, trans


@torch.no_grad()
def gdrn_inference_on_dataset(cfg, model, datasets_root, *, train_obj_ids=None, max_batch=None, num_workers=8,
                              use_cuda_graph=True, device="cuda", test_set=None, stats=None):
    """Run the test loop: -> records [{scene_id, im_id, obj_id, score, R [3,3], t [3] metres, time}] in image order,
    then ROI order.  model: a GDRN_DoubleMask built from cfg, or a PerObjectGDRN keyed by label.  train_obj_ids: the
    objects a per-object checkpoint covers (ROIs of other objects are dropped).  stats: a dict that receives the
    per-stage times (seconds): decode (host, summed over threads), h2d / roi_build / forward / post / d2h (device
    events), wall, and the batch count."""
    device = torch.device(device)
    ts = test_set or TestSet(cfg, datasets_root, train_obj_ids)
    with_depth = bool(cfg_get(cfg, "TEST.USE_DEPTH_REFINE", False)) and not cfg_get(cfg, "TEST.USE_PNP", False)
    meshes = ts.meshes(device) if with_depth else None
    mask_thr = float(cfg_get(cfg, "MODEL.POSE_NET.GEO_HEAD.MASK_THR_TEST", 0.5))
    return _run_batches(cfg, model, ts, _PoseRows(cfg, ts, meshes, mask_thr), with_depth, max_batch, num_workers,
                        use_cuda_graph, device, stats)


class _PoseRows:
    """Output step of the test loop: GDRN_Evaluator.process's post-processing dispatch, one D2H copy of the poses, one
    result row per ROI."""

    def __init__(self, cfg, ts, meshes, mask_thr):
        self.cfg, self.ts, self.meshes, self.mask_thr = cfg, ts, meshes, mask_thr
        self.pose_dev = {}

    def post(self, inp, out, n, slot, hw):
        rot, trans = postprocess(self.cfg, inp, out, self.meshes, self.mask_thr)
        pose = self.pose_dev.get(n)
        if pose is None:
            pose = self.pose_dev[n] = torch.empty((n, 3, 4), dtype=torch.float32, device=rot.device)
        pose[:, :, :3].copy_(rot)
        pose[:, :, 3].copy_(trans)
        return pose

    def d2h(self, pose):
        host_pose = torch.empty(tuple(pose.shape), dtype=torch.float32, pin_memory=True)
        host_pose.copy_(pose, non_blocking=True)
        return host_pose

    def empty(self):
        return torch.empty((0, 3, 4))

    def rows(self, imgs, host_pose, batch_seconds):
        return batch_rows(self.ts.images, imgs, host_pose.numpy(), batch_seconds)


def _run_batches(cfg, model, ts, output, with_depth, max_batch, num_workers, use_cuda_graph, device, stats):
    """The batched loop shared by the test and save-results loops; ``output`` is the per-batch output step:
    post(inp, out, n, slot, (H, W)) enqueues its device work after the forward (slot: the batch's double-buffer index),
    d2h(state) enqueues the copies to the host, and rows(imgs, payload, batch_seconds) turns them into results once the
    batch's copies are done (empty() is the payload of a batch without ROIs)."""
    if not isinstance(model, PerObjectGDRN) and model.class_aware and model.num_classes != len(ts.obj_ids):
        raise ValueError(f"MODEL.POSE_NET.NUM_CLASSES={model.num_classes} but dataset {ts.dataset!r} has "
                         f"{len(ts.obj_ids)} objects")
    if max_batch is None:
        max_batch = max(m.max_batch for m in model.members.values()) if isinstance(model, PerObjectGDRN) else model.max_batch
    in_res, out_res = cfg_get(cfg, "MODEL.POSE_NET.INPUT_RES", 256), cfg_get(cfg, "MODEL.POSE_NET.OUTPUT_RES", 64)
    pix_mean, pix_std = cfg_get(cfg, "MODEL.PIXEL_MEAN", (0.0, 0.0, 0.0)), cfg_get(cfg, "MODEL.PIXEL_STD", (255.0, 255.0, 255.0))
    dzi = float(cfg_get(cfg, "INPUT.DZI_PAD_SCALE", 1.5))
    records = ts.records
    if not records:
        return []
    keys = [image_shape(ts.rgb[i]) for i, _ in records]   # file headers only; batches hold images of one shape
    for shape in sorted(set(keys)):
        check_config(cfg, shape[:2])
    batches = pack_batches([len(a) for _, a in records], max_batch, keys)
    static, graphs = {}, {}
    stages = [_Stage(device), _Stage(device)]
    stream = torch.cuda.current_stream(device)
    timing = stats is not None
    ev = lambda: torch.cuda.Event(enable_timing=True)
    dec_time = [0.0]
    lock = threading.Lock()

    def fill(stage, batch):
        """Decode one batch straight into the stage's pinned block (runs on the pool)."""
        imgs = [records[p] for p in batch]
        N = len(imgs)
        H, W, C = keys[batch[0]]
        n = sum(len(a) for _, a in imgs)
        stage.layout(N, H, W, C, n, with_depth)
        h = stage.h

        def one(j):
            t0 = time.perf_counter()
            idx = imgs[j][0]
            im = read_image(ts.rgb[idx])
            if im.shape != (H, W, C):
                raise ValueError(f"{ts.rgb[idx]}: {im.shape} in a batch of {(H, W, C)} images")
            h["images"][j].numpy()[...] = im
            if with_depth:
                h["depth"][j].numpy()[...] = read_depth(ts.depth[idx])
            with lock:
                dec_time[0] += time.perf_counter() - t0

        list(pool.map(one, range(N)))
        h["K"].numpy()[...] = np.stack([ts.K[i] for i, _ in imgs])
        if with_depth:
            h["depth_factor"].numpy()[...] = [ts.depth_factor[i] for i, _ in imgs]
        meta = [(j, a["label"]) for j, (_, anns) in enumerate(imgs) for a in anns]
        xywh = [a["bbox_est"] for _, anns in imgs for a in anns]
        if n:
            h["det_meta"].numpy()[...] = np.asarray(meta, np.int32)
            h["bbox_est"].numpy()[...] = np.asarray(xywh, np.float32)   # torch.tensor(list) in BoxMode.convert: float32
        return imgs, n

    out_rows = []
    pending = None   # the previous batch: (imgs, payload of its D2H copies, event after them)
    tstat = {"h2d": [], "roi_build": [], "forward": [], "post": [], "d2h": []}
    pool = ThreadPoolExecutor(num_workers)
    feeder = ThreadPoolExecutor(1)
    t_start = time.perf_counter()
    t_last = [t_start]

    def finish(p):
        imgs, payload, done = p
        done.synchronize()
        now = time.perf_counter()
        out_rows.extend(output.rows(imgs, payload, now - t_last[0]))
        t_last[0] = now

    try:
        fut = feeder.submit(fill, stages[0], batches[0])
        for bi in range(len(batches)):
            stage = stages[bi % 2]
            imgs, n = fut.result()
            if bi + 1 < len(batches):
                nxt = stages[(bi + 1) % 2]
                if nxt.h2d_done is not None:
                    nxt.h2d_done.synchronize()   # its pinned block was last copied by batch bi - 1
                fut = feeder.submit(fill, nxt, batches[bi + 1])
            e = [ev() for _ in range(6)] if timing else None
            if timing:
                e[0].record(stream)
            stage.dev[:stage.nbytes].copy_(stage.host[:stage.nbytes], non_blocking=True)
            stage.h2d_done = torch.cuda.Event()
            stage.h2d_done.record(stream)
            if timing:
                e[1].record(stream)
            if n == 0:
                payload = output.empty()
                done = torch.cuda.Event()
                done.record(stream)
            else:
                st = static.get((n, with_depth))
                if st is None:
                    st = static[(n, with_depth)] = roi_batch_buffers(n, device, in_res, out_res, with_depth)
                d = stage.d
                inp = roi_batch_inputs(d["images"], {"det_meta": d["det_meta"], "bbox_est": d["bbox_est"]}, d["K"],
                                       ts.extents(device), dzi, in_res, out_res, pix_mean, pix_std,
                                       depth=d["depth"] if with_depth else None,
                                       depth_factor=d["depth_factor"] if with_depth else None, out=st)
                if timing:
                    e[2].record(stream)
                out = _forward(model, inp, graphs, use_cuda_graph)
                if timing:
                    e[3].record(stream)
                state = output.post(inp, out, n, bi % 2, keys[batches[bi][0]][:2])
                if timing:
                    e[4].record(stream)
                payload = output.d2h(state)
                done = torch.cuda.Event()
                done.record(stream)
                if timing:
                    e[5].record(stream)
                    for k, (a, b) in zip(("h2d", "roi_build", "forward", "post", "d2h"), zip(e[:-1], e[1:])):
                        tstat[k].append((a, b))
            if pending is not None:
                finish(pending)
            pending = (imgs, payload, done)
        if pending is not None:
            finish(pending)
    finally:
        pool.shutdown()
        feeder.shutdown()
    if timing:
        torch.cuda.synchronize(device)
        stats.update({k: sum(a.elapsed_time(b) for a, b in v) / 1e3 for k, v in tstat.items()})
        stats["decode"] = dec_time[0]
        stats["wall"] = time.perf_counter() - t_start
        stats["batches"] = len(batches)
        stats["images"] = len(records)
        stats["rois"] = sum(len(a) for _, a in records)
    return out_rows


def batch_rows(images, imgs, poses, batch_seconds):
    """Result rows of one batch: imgs [(image index, dets)], poses [n,3,4] in ROI order.  An image's time is its
    detection time (its first ROI's, gdrn_evaluator.py:754-760) plus batch_seconds / number of images in the batch."""
    share = batch_seconds / max(len(imgs), 1)
    rows, k = [], 0
    for idx, anns in imgs:
        sid, iid = images[idx]
        t_img = (anns[0]["time"] if anns else 0.0) + share
        for a in anns:
            rows.append({"scene_id": sid, "im_id": iid, "obj_id": a["obj_id"], "score": float(np.float32(a["score"])),
                         "R": poses[k, :, :3].astype(np.float64), "t": poses[k, :, 3].astype(np.float64), "time": t_img})
            k += 1
    return rows


# ------------------------------------------------------------------------------------------------ save results
def save_record(det, pose, mask_rle, full_mask_rle, use_pnp):
    """One ROI's entry of results.pkl (gdrn_save_result_of_dataset, gdrn_evaluator.py:957-976): bbox_est is the
    loader's float32 XYXY box; R / t are the network's float32 pose, or with TEST.USE_PNP misc.pnp_v2's float64 pose
    (the float32 -100 sentinel where fewer than 4 points were selected)."""
    x, y, w, h = np.asarray(det["bbox_est"], np.float32)
    pose = np.asarray(pose, np.float32)
    if use_pnp and not (pose == -100).all():
        pose = pose.astype(np.float64)
    return {"obj_id": det["obj_id"], "score": float(np.float32(det["score"])),
            "bbox_est": np.array([x, y, x + w, y + h], np.float32), "mask": mask_rle, "full_mask": full_mask_rle,
            "R": pose[:, :3].copy(), "t": pose[:, 3].copy()}


class _SaveRecords:
    """Output step of the save-results loop: the pose (TEST.USE_PNP: get_pnp_ransac_pose, i.e. pnp_ransac_from_maps;
    else the network's; never depth refine) and both masks pasted and RLE-encoded on the device (gdrn_mask_paste_rle).
    The [2n,2] string table travels with the poses; the string bytes follow in rows(), after the batch's event, from
    this slot's device buffer (two slots: batch k + 1 is already running when batch k's strings are copied)."""

    def __init__(self, cfg, ts, mask_thr, device):
        from .native_ops import MaskRleBuffers, mask_prob_mode

        self.ts, self.mask_thr = ts, mask_thr
        self.use_pnp = bool(cfg_get(cfg, "TEST.USE_PNP", False))
        # both masks use MASK_LOSS_TYPE, as get_out_mask(cfg, ...) does for the full mask too
        self.loss_type = str(cfg_get(cfg, "MODEL.POSE_NET.LOSS_CFG.MASK_LOSS_TYPE", "L1"))
        mask_prob_mode(self.loss_type)
        self.bufs = [MaskRleBuffers(device), MaskRleBuffers(device)]
        self.pose_dev = {}
        self.side = torch.cuda.Stream(device)
        self.host_chars = torch.empty(0, dtype=torch.uint8).pin_memory()

    def post(self, inp, out, n, slot, hw):
        from .native_ops import paste_masks_rle_launch

        pose = self.pose_dev.get(n)
        if pose is None:
            pose = self.pose_dev[n] = torch.empty((n, 3, 4), dtype=torch.float32, device=out["rot"].device)
        if self.use_pnp:
            from .pnp_ransac import pnp_ransac_from_maps

            pose.copy_(pnp_ransac_from_maps(out["coor_x"], out["coor_y"], out["coor_z"], out["mask"], inp["roi_coord_2d"],
                                            inp["im_H"], inp["im_W"], inp["roi_extent"], inp["roi_cam"],
                                            mask_thr=self.mask_thr))
        else:
            pose[:, :, :3].copy_(out["rot"])
            pose[:, :, 3].copy_(out["trans"])
        bufs = paste_masks_rle_launch(out["mask"], out["full_mask"], inp["roi_center"], inp["scale"], hw, self.mask_thr,
                                      self.loss_type, self.bufs[slot])
        return pose, bufs, n, hw

    def d2h(self, state):
        pose, bufs, n, hw = state
        host_pose = torch.empty((n, 3, 4), dtype=torch.float32, pin_memory=True)
        host_pose.copy_(pose, non_blocking=True)
        host_table = torch.empty((2 * n, 2), dtype=torch.int64, pin_memory=True)
        host_table.copy_(bufs.table[:2 * n], non_blocking=True)
        return host_pose, host_table, bufs, hw

    def empty(self):
        return None

    def rows(self, imgs, payload, batch_seconds):
        if payload is None:
            return []
        from .native_ops import rle_dicts

        host_pose, host_table, bufs, (H, W) = payload
        table = host_table.numpy()
        total = int(table[-1].sum())
        if self.host_chars.numel() < total:
            self.host_chars = torch.empty(total, dtype=torch.uint8).pin_memory()
        with torch.cuda.stream(self.side):   # the batch's kernels are done (its event was waited on)
            self.host_chars[:total].copy_(bufs.chars[:total], non_blocking=True)
        self.side.synchronize()
        rles = rle_dicts(table, self.host_chars[:total].numpy(), H, W)
        n = len(rles) // 2
        poses = host_pose.numpy()
        out, k = [], 0
        for idx, anns in imgs:
            sid, iid = self.ts.images[idx]
            for a in anns:
                out.append((f"{sid}/{iid}", save_record(a, poses[k], rles[k], rles[n + k], self.use_pnp)))
                k += 1
        return out


def save_results_dir(cfg, per_object=False):
    """do_save_results's directory (engine/engine.py:121-131): <OUTPUT_DIR>/inference_<basename(MODEL.WEIGHTS) up to its
    first ".">/<DATASETS.TEST[0]>; per_object (several per-object checkpoints in one run): inference_per_object."""
    tests = list(cfg_get(cfg, "DATASETS.TEST", ()) or ())
    if len(tests) != 1:
        raise ValueError(f"DATASETS.TEST={tests!r}: the save-results loop writes one dataset's results.pkl; "
                         "give exactly one DATASETS.TEST entry")
    model_name = "per_object" if per_object else os.path.basename(str(cfg_get(cfg, "MODEL.WEIGHTS", ""))).split(".")[0]
    return os.path.join(str(cfg_get(cfg, "OUTPUT_DIR", "output")), f"inference_{model_name}", tests[0])


def write_results_pkl(result, output_dir):
    """mmcv.dump(result, <dir>/results.pkl): pickle protocol 2."""
    import pickle

    os.makedirs(output_dir, exist_ok=True)
    path = os.path.join(output_dir, "results.pkl")
    with open(path, "wb") as f:
        pickle.dump(result, f, protocol=2)
    return path


@torch.no_grad()
def gdrn_save_result_of_dataset(cfg, model, datasets_root, output_dir, *, train_obj_ids=None, max_batch=None,
                                num_workers=8, use_cuda_graph=True, device="cuda", test_set=None, stats=None):
    """The save-results loop (save_gdrn.sh -> TEST.SAVE_RESULTS_ONLY -> gdrn_save_result_of_dataset,
    gdrn_evaluator.py:812-1119) on the batching, decode pool, ROI build, CUDA graphs and D2H pipeline of the test loop.
    -> {"scene_id/im_id": [{obj_id, score, bbox_est, mask, full_mask, R, t}, ...]} in image order, then ROI order (an
    image without ROIs has no key), also written to <output_dir>/results.pkl.  model must return the geometry maps
    (built from a config with TEST.SAVE_RESULTS_ONLY=True or TEST.USE_PNP=True)."""
    if not model.wants_maps:
        raise ValueError("gdrn_save_result_of_dataset needs the mask maps: build the model from a config with "
                         "TEST.SAVE_RESULTS_ONLY=True")
    device = torch.device(device)
    ts = test_set or TestSet(cfg, datasets_root, train_obj_ids)
    mask_thr = float(cfg_get(cfg, "MODEL.POSE_NET.GEO_HEAD.MASK_THR_TEST", 0.5))
    rows = _run_batches(cfg, model, ts, _SaveRecords(cfg, ts, mask_thr, device), False, max_batch, num_workers,
                        use_cuda_graph, device, stats)
    result = results_dict(rows)
    write_results_pkl(result, output_dir)
    return result


def results_dict(rows):
    """[("scene_id/im_id", record), ...] in image order, then ROI order -> {key: [record, ...]} in the same order."""
    result = {}
    for key, rec in rows:
        result.setdefault(key, []).append(rec)
    return result


# ------------------------------------------------------------------------------------------------ results
class GdrnDatasetEvaluator:
    """Writes the results CSV (save_and_eval_results) and, unless VAL.SAVE_BOP_CSV_ONLY, scores it in-process with
    eval_pose_results_more.run, passing the arguments save_and_eval_results passes to VAL.SCRIPT_PATH."""

    def __init__(self, cfg, datasets_root, output_dir, exp_id_str):
        self.cfg = cfg
        self.datasets_root = datasets_root
        self.output_dir = output_dir
        self.exp_id = exp_id_str

    def evaluate(self, records):
        cfg = self.cfg
        os.makedirs(self.output_dir, exist_ok=True)
        name = result_csv_name(cfg, self.exp_id)
        bop_eval.write_bop_results_csv(records, os.path.join(self.output_dir, name))
        if cfg_get(cfg, "VAL.SAVE_BOP_CSV_ONLY", False):
            return {"csv": os.path.join(self.output_dir, name)}
        from . import eval_pose_results_more as E

        argv = ["--results_path", self.output_dir, "--result_filenames", name,
                "--renderer_type", str(cfg_get(cfg, "VAL.RENDERER_TYPE", "cpp")),
                "--error_types", str(cfg_get(cfg, "VAL.ERROR_TYPES", E.DEFAULT_ERROR_TYPES)),
                "--eval_path", self.output_dir, "--targets_filename", str(cfg_get(cfg, "VAL.TARGETS_FILENAME")),
                "--n_top", str(cfg_get(cfg, "VAL.N_TOP", -1)),
                "--datasets_path", os.path.join(self.datasets_root, "BOP_DATASETS")]
        if cfg_get(cfg, "VAL.SCORE_ONLY", False):
            argv.append("--score_only")
        scores = E.run(E.parse_args(argv))
        final = scores[os.path.splitext(name)[0]]
        print("scores_bop19:", json.dumps({k: float(v) for k, v in sorted(final.items())}))
        return {"csv": os.path.join(self.output_dir, name), "scores": final}


def build_model(cfg, weights, *, obj_ids=None, precision=None, max_batch=64, device="cuda", use_cuda_graph=True):
    """GDRN_DoubleMask from cfg + one checkpoint (path or state_dict), or with weights = {obj_id: ckpt} one class-agnostic
    member per object behind PerObjectGDRN (labels from obj_ids, the dataset's label table)."""
    from .gdrn_model import GDRN_DoubleMask
    from .predictor import _arch

    def load(w):
        if isinstance(w, Mapping):
            return w
        ck = torch.load(w, map_location="cpu")
        sd = ck.get("model", ck)
        return {k[len("_module."):] if k.startswith("_module.") else k: v for k, v in sd.items()}

    def one(w):
        m = GDRN_DoubleMask(cfg, arch=_arch(cfg), max_batch=max_batch, precision=precision)
        m.load_state_dict(load(w))
        return m.to(device)

    per_object = isinstance(weights, Mapping) and weights and all(
        isinstance(k, int) or str(k).isdigit() for k in weights) and not all(torch.is_tensor(v) for v in weights.values())
    if per_object:
        if obj_ids is None:
            raise ValueError("per-object weights need the dataset's label table (obj_ids)")
        return PerObjectGDRN({obj_ids.index(int(k)): one(v) for k, v in weights.items()}, use_cuda_graph=use_cuda_graph)
    return one(weights)
