"""The xyz_crop training targets of a BOP split as batched GPU passes (the reference's *_1_gen_xyz.py scripts).

Mirrors, without a GL context:
  * core/gdrn_modeling/tools/{icbin,itodd,tudl}/*_pbr_1_gen_xyz.py
  * core/gdrn_modeling/tools/tless/tless_{pbr,primesense}_1_gen_xyz.py
Every entry of every image's scene_gt.json gets <xyz_root>/<scene:06d>/<im:06d>_<anno_i:06d>-xyz.pkl, the pickle
(protocol 2) of {"xyz_crop": float16 [h,w,3], "xyxy": [x1, y1, x2, y2]}: the instance rendered alone, back-projected to
model coordinates (misc.calc_xyz_bp_torch) and cropped to the inclusive box of its coverage.  An instance that renders
to nothing gets full-frame zeros and the box [0, 0, W - 1, H - 1].  The data loader (data_loader.py, XYZ_ONLINE=False)
reads these files through each registrar's xyz_path.

The renders come from the CUDA rasteriser (renderer.render_meshes, float z); two kernels (csrc/xyz_crop.cu) find the
boxes and pack the fp16 crops of many instances.  No CPU fallback: the GPU path needs CUDA and raises GdrnError
otherwise.

  python -m gdrnpp_bop2022_b200.gen_xyz --dataset tless --dataset_split train --dataset_split_type pbr
"""
import argparse
import json
import os
import pickle
import sys
import time
from concurrent.futures import ThreadPoolExecutor

if __package__ in (None, ""):   # run by path
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    __package__ = "gdrnpp_bop2022_b200"

import numpy as np
import torch

from . import _lib
from . import gt_info
from ._lib import GdrnError

DEFAULT_MAX_BYTES = 2 << 30
ZNEAR, ZFAR = 0.01, 6.5       # the scripts' near / far, the same in all of them
VERTEX_SCALE = 0.001          # models in mm, rendered in metres
RENDER_BYTES_PER_PIXEL = 12   # render_meshes: f32 depth + the rasteriser's 64-bit z-buffer


def xyz_path(xyz_root, scene_id, im_id, anno_i):
    """The file of one GT entry, as the scripts write it and the registrars' xyz_path reads it."""
    return os.path.join(xyz_root, "{:06d}".format(scene_id), "{:06d}_{:06d}-xyz.pkl".format(im_id, anno_i))


def dumps(xyz_crop, xyxy):
    """The file's bytes: mmcv.dump(dict, path) of a .pkl is pickle protocol 2, keys in this order."""
    return pickle.dumps({"xyz_crop": xyz_crop, "xyxy": [int(v) for v in xyxy]}, protocol=2)


# ---------------------------------------------------------------------------------------------------------------------
# In-memory API
def _f32(a, shape):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32).reshape(shape)))


class _HostBuf:
    """One growable host buffer of fp16 crops: chunks land back to back; growing keeps what has already landed."""

    def __init__(self, staging=None, slot=0):
        self.staging, self.slot = staging, slot
        self.buf = None if staging is None else staging.slots[slot]
        self.used = 0

    def reserve(self, numel):
        need = self.used + numel
        if self.buf is None or self.buf.numel() < need or self.buf.dtype != torch.float16:
            cap = max(need, 2 * (self.buf.numel() if self.buf is not None and self.buf.dtype == torch.float16 else 0))
            nb = torch.empty(max(cap, 1), dtype=torch.float16, pin_memory=torch.cuda.is_available())
            if self.used:
                nb[:self.used].copy_(self.buf[:self.used])
            self.buf = nb
            if self.staging is not None:
                self.staging.slots[self.slot] = nb
        view = self.buf[self.used:need]
        self.used = need
        return view


def crops_async(models, obj_index, R, t, K, H, W, znear=ZNEAR, zfar=ZFAR, max_bytes=DEFAULT_MAX_BYTES, staging=None,
                slot=0):
    """Run the crops of n instances of H x W images into pinned host memory; the caller waits on the returned event.
    models: renderer.Model3D list (metres); obj_index [n] indexes it; R [n,3,3], t [n,3] (metres), K [n,3,3], all
    taken as f32.  Instances go through the renders in chunks whose renders fit max_bytes (12 B per pixel); each
    chunk costs two device-to-host copies, its boxes (which size its packed buffer) and its packed crops.
    staging / slot: a gt_info._Staging whose slot holds the host buffer (reused and grown as needed).
    -> (boxes [n,4] i64 x1, y1, x2, y2 (full frame for an empty instance), empty [n] bool, offsets [n+1] i64 in fp16
    elements of the host buffer, host buffer f16, CUDA event of the last copy or None)."""
    from . import renderer

    n = len(obj_index)
    dev = models[0].vertices.device if models else torch.device("cuda")
    host = _HostBuf(staging, slot)
    boxes = np.zeros((n, 4), np.int64)
    empty_all = np.zeros(n, bool)
    offsets = np.zeros(n + 1, np.int64)
    if n == 0:
        return boxes, empty_all, offsets, host.reserve(0), None
    with torch.cuda.device(dev):
        idx = np.asarray(obj_index, np.int64).reshape(n)
        if idx.min() < 0 or idx.max() >= len(models):
            raise GdrnError("gen_xyz: obj_index out of range [0, {})".format(len(models)))
        reg = np.array([m.mesh_id for m in models], np.int32)
        ids = torch.from_numpy(reg[idx]).to(dev)
        Rt, tt, Kt = _f32(R, (n, 3, 3)), _f32(t, (n, 3, 1)), _f32(K, (n, 3, 3))
        poses = torch.cat([Rt, tt], dim=2).to(dev)
        Rd, td, Kd = Rt.reshape(n, 9).to(dev), tt.reshape(n, 3).to(dev), Kt.reshape(n, 9).to(dev)
        chunk = max(1, int(max_bytes) // (RENDER_BYTES_PER_PIXEL * H * W))
        L = _lib.lib()
        stream = _lib.current_stream()
        base = 0
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            c = e - s
            depth = renderer.render_meshes(ids[s:e], poses[s:e], Kd[s:e], H, W, znear, zfar)
            d_boxes = torch.empty((c, 4), dtype=torch.int32, device=dev)
            _lib.check(L.gdrn_xyz_crop_boxes(_lib.ptr(depth), c, H, W, _lib.ptr(d_boxes), stream), "gdrn_xyz_crop_boxes")
            b = d_boxes.cpu().numpy().astype(np.int64)     # copy 1: the boxes size the packed buffer
            empty = b[:, 0] > b[:, 2]
            b[empty] = (0, 0, W - 1, H - 1)
            sizes = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1) * 3
            offs = np.zeros(c + 1, np.int64)
            np.cumsum(sizes, out=offs[1:])
            boxes[s:e] = b
            empty_all[s:e] = empty
            offsets[s + 1:e + 1] = base + offs[1:]
            out = torch.empty(max(int(offs[-1]), 1), dtype=torch.float16, device=dev)
            d_offs = torch.from_numpy(offs[:c]).to(dev)
            _lib.check(L.gdrn_xyz_crop_pack(_lib.ptr(depth), _lib.ptr(Rd[s:e]), _lib.ptr(td[s:e]), _lib.ptr(Kd[s:e]),
                                            _lib.ptr(d_boxes), _lib.ptr(d_offs), c, H, W, _lib.ptr(out), stream),
                       "gdrn_xyz_crop_pack")
            host.reserve(int(offs[-1])).copy_(out[:int(offs[-1])], non_blocking=True)   # copy 2: the packed crops
            base += int(offs[-1])
        ev = torch.cuda.Event()
        ev.record()
    return boxes, empty_all, offsets, host.buf[:base], ev


def split_crops(boxes, offsets, host, H, W):
    """The per-instance results of crops_async: [(xyxy, float16 [h,w,3] view of host)]."""
    h = host.numpy() if torch.is_tensor(host) else host
    out = []
    for i in range(len(boxes)):
        x1, y1, x2, y2 = (int(v) for v in boxes[i])
        out.append(([x1, y1, x2, y2], h[offsets[i]:offsets[i + 1]].reshape(y2 - y1 + 1, x2 - x1 + 1, 3)))
    return out


def xyz_crops(models, obj_index, R, t, K, H, W, znear=ZNEAR, zfar=ZFAR, max_bytes=DEFAULT_MAX_BYTES):
    """The xyz_crop of n instances of H x W images, each rendered alone (see crops_async for the arguments).
    -> [(xyxy [x1, y1, x2, y2] ints, float16 [y2-y1+1, x2-x1+1, 3])]; an instance that renders to nothing gets
    [0, 0, W - 1, H - 1] and zeros."""
    boxes, _, offsets, host, ev = crops_async(models, obj_index, R, t, K, H, W, znear, zfar, max_bytes)
    if ev is not None:
        ev.synchronize()
    return split_crops(boxes, offsets, host, H, W)


# ---------------------------------------------------------------------------------------------------------------------
# Split driver: plan every GT entry, drop those already written, then per batch of images of one scene one GPU pass
# (crops_async) while the previous batch's pickles are written on a thread pool
def image_size(path):
    """(H, W) of an image from its header."""
    from PIL import Image

    with Image.open(path) as im:
        return im.size[1], im.size[0]


def plan(sp, xyz_root, scene_ids=None):
    """-> [(scene_id, H, W, [(im_id, [instance records])])] of the instances still to write, and the number of GT
    entries skipped because their file exists with size > 0 (the scripts' resume rule).  Instance record = {anno_i,
    obj_id, R [3,3] f32, t [3] f32 in metres (cam_t_m2c / 1000 in f32), K [3,3] f32, path}.  The image size of a scene
    is its colour images' size; rejects a missing colour image or a scene of mixed sizes before any work."""
    scenes, skipped = [], 0
    for scene_id, ims in gt_info.plan_split(sp, scene_ids, need_depth=False):
        size, todo = None, []
        for im in ims:
            p = gt_info.image_path(sp, scene_id, im["im_id"])
            hw = image_size(p)
            if size is None:
                size, first = hw, p
            elif hw != size:
                raise GdrnError("image {} is {}x{}, {} of the same scene is {}x{}".format(p, hw[1], hw[0], first, size[1],
                                                                                        size[0]))
            K = np.asarray(im["K"], np.float32).reshape(3, 3)
            insts = []
            for anno_i, g in enumerate(im["gts"]):
                path = xyz_path(xyz_root, scene_id, im["im_id"], anno_i)
                if os.path.exists(path) and os.path.getsize(path) > 0:
                    skipped += 1
                    continue
                insts.append({"anno_i": anno_i, "obj_id": int(g["obj_id"]),
                              "R": np.asarray(g["cam_R_m2c"], np.float32).reshape(3, 3),
                              "t": np.asarray(g["cam_t_m2c"], np.float32).reshape(3) / np.float32(1000.0), "K": K,
                              "path": path})
            if insts:
                todo.append((im["im_id"], insts))
        scenes.append((scene_id, size, todo, len(ims)))
    return scenes, skipped


def load_models(model_dir, obj_ids, device="cuda"):
    """{obj_id: renderer.Model3D} of the models the instances use, scaled to metres as the scripts' EGLRenderer
    (vertex_scale=0.001) scales them; rejects an obj_id without a model file."""
    from . import renderer

    return {o: renderer.Model3D(pts * VERTEX_SCALE, faces, device=device)
            for o, (pts, faces) in gt_info.load_models(model_dir, obj_ids).items()}


def _write(path, xyz_crop, xyxy):
    """One file, written whole under a temporary name and then renamed, so that an interrupted run leaves no partial
    file that the resume rule would take for a finished one."""
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        f.write(dumps(xyz_crop, xyxy))
    os.replace(tmp, path)


def run_split(sp, model_dir, xyz_root=None, scene_ids=None, max_bytes=DEFAULT_MAX_BYTES, batch_images=16, workers=8,
              device="cuda", log=print, models=None):
    """Write the xyz_crop file of every GT entry of a split that does not have one yet.  xyz_root defaults to
    <split_path>/xyz_crop.  models: {obj_id: renderer.Model3D} to reuse (default: loaded from model_dir).  log: called
    with one line per instance that renders to nothing (and so gets full-frame zeros).
    -> {"images", "written", "skipped", "empty", "seconds"}."""
    t0 = time.time()
    xyz_root = os.path.join(sp["split_path"], "xyz_crop") if xyz_root is None else xyz_root
    scenes, skipped = plan(sp, xyz_root, scene_ids)
    used = {i["obj_id"] for _, _, todo, _ in scenes for _, insts in todo for i in insts}
    if models is None or not used <= set(models):
        models = load_models(model_dir, used, device)
    order = sorted(models)
    model_list = [models[o] for o in order]
    index = {o: k for k, o in enumerate(order)}
    step = max(1, int(batch_images))
    batches = [(scene_id, size, todo[k:k + step]) for scene_id, size, todo, _ in scenes for k in range(0, len(todo), step)]
    staging = gt_info._Staging()
    pool = ThreadPoolExecutor(max(1, workers))
    slot_writes = [[], []]
    n_written = n_empty = 0

    def finish(p):
        nonlocal n_written, n_empty
        (scene_id, (H, W), ims), (boxes, empty, offsets, host, ev), k = p
        if ev is not None:
            ev.synchronize()
        insts = [(im_id, inst) for im_id, insts in ims for inst in insts]
        for i, (xyxy, crop) in enumerate(split_crops(boxes, offsets, host, H, W)):
            im_id, inst = insts[i]
            if empty[i]:
                n_empty += 1
                if log:
                    log("not visible: scene {} image {} entry {} obj_id {}".format(scene_id, im_id, inst["anno_i"],
                                                                                   inst["obj_id"]))
            slot_writes[k].append(pool.submit(_write, inst["path"], crop, xyxy))
        n_written += len(insts)

    try:
        for scene_id, _, todo, _ in scenes:
            if todo:
                os.makedirs(os.path.join(xyz_root, "{:06d}".format(scene_id)), exist_ok=True)
        pending = None
        for b, (scene_id, (H, W), ims) in enumerate(batches):
            k = b % 2
            for f in slot_writes[k]:   # the host slot is reused: its earlier writes must be done
                f.result()
            slot_writes[k] = []
            insts = [inst for _, insts in ims for inst in insts]
            res = crops_async(model_list, [index[i["obj_id"]] for i in insts], np.stack([i["R"] for i in insts]),
                              np.stack([i["t"] for i in insts]), np.stack([i["K"] for i in insts]), H, W, ZNEAR, ZFAR,
                              max_bytes, staging, k)
            if pending is not None:
                finish(pending)
            pending = ((scene_id, (H, W), ims), res, k)
        if pending is not None:
            finish(pending)
        for fs in slot_writes:
            for f in fs:
                f.result()
    finally:
        pool.shutdown(wait=True)
    return {"images": sum(n for *_, n in scenes), "written": n_written, "skipped": skipped, "empty": n_empty,
            "seconds": time.time() - t0}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="xyz_crop training targets of a BOP split on the GPU (the *_1_gen_xyz.py "
                                             "scripts)")
    ap.add_argument("--dataset", required=True)
    ap.add_argument("--dataset_split", default="train")
    ap.add_argument("--dataset_split_type", default=None)
    ap.add_argument("--datasets_path", default=os.environ.get("BOP_PATH", "datasets/BOP_DATASETS/"))
    ap.add_argument("--models_dir", default=None, help="directory of obj_XXXXXX.ply (default: as the scripts pick)")
    ap.add_argument("--model_type", default=None, help="models_<model_type>/ (T-LESS primesense: reconst)")
    ap.add_argument("--xyz_root", default=None, help="output directory (default: <split_path>/xyz_crop)")
    ap.add_argument("--scene_ids", default=None, help="comma-separated scene ids (default: every scene of the split)")
    ap.add_argument("--max_bytes", default=DEFAULT_MAX_BYTES, type=int, help="device memory budget of one render chunk")
    ap.add_argument("--batch_images", default=16, type=int, help="images per batch")
    args = ap.parse_args(argv)
    if args.models_dir and args.model_type:
        ap.error("give --models_dir or --model_type, not both")
    if args.scene_ids is not None:
        args.scene_ids = [int(s) for s in args.scene_ids.split(",") if s]
    return args


def resolve(args):
    """-> (split params, model directory, xyz_root) of parsed arguments."""
    sp = gt_info.split_params(args.datasets_path, args.dataset, args.dataset_split, args.dataset_split_type)
    model_dir = gt_info.models_path(args.datasets_path, args.dataset, args.models_dir, args.model_type)
    return sp, model_dir, args.xyz_root or os.path.join(sp["split_path"], "xyz_crop")


def main(argv=None):
    args = parse_args(argv)
    sp, model_dir, xyz_root = resolve(args)
    r = run_split(sp, model_dir, xyz_root, args.scene_ids, args.max_bytes, args.batch_images)
    print(json.dumps({"split_path": sp["split_path"], "xyz_root": xyz_root, **r}))
    return r


if __name__ == "__main__":
    main()
