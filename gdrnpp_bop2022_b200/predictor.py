"""GdrnPredictor -- the single-image API of the reference (core/gdrn_modeling/demo/predictor_gdrn.py:44-476),
routed to the CUDA hot path.

Same constructor signature, method names and data contracts as the reference:
``GdrnPredictor(config_file_path, ckpt_file_path, camera_json_path, path_to_obj_models)``;
``preprocessing(outputs, image, depth_img) -> data_dict``, ``inference(data_dict) -> out_dict``,
``postprocessing(data_dict, out_dict) -> {obj_name: 4x4 pose}``, ``process_depth_refine(data_dict, out_dict)``.
Keyword-only extras let a caller hand over already-loaded pieces instead of paths (``state_dict``, ``cam``, ``objs``,
``extents``, ``models``) -- there are no datasets or checkpoints in this environment, so the tests use those.
``inference`` and ``process_depth_refine`` run entirely in libgdrn_b200.so; ``preprocessing`` crops the ROIs with the
batched GPU restatement of cv2.warpAffine (crop_resize_by_warp_affine, SURVEY.md §8f rank 1); ``postprocessing`` with
``TEST.USE_PNP`` (the reference predictor's default, predictor_gdrn.py:58) runs the batched GPU RANSAC-PnP
(``pnp_ransac.py``) instead of the per-ROI ``cv2.solvePnPRansac`` loop (engine/gdrn_evaluator.py:1122-1221).
"""
import glob
import json
import os
import re
from collections.abc import Mapping

import numpy as np
import torch

from .gdrn_model import GDRN_DoubleMask, _cfg_get, default_cfg, load_py_config
from .native_ops import crop_resize_float, crop_resize_image, get_affine_transform
from .per_object import PerObjectGDRN
from .ply import load_ply
from .renderer import Model3D, depth_refine, get_K_crop_resize


class GdrnPredictor:
    def __init__(self, config_file_path=None, ckpt_file_path=None, camera_json_path=None, path_to_obj_models=None, *,
                 cam=None, objs=None, extents=None, models=None, state_dict=None, num_classes=None, cfg=None,
                 use_pnp=None, use_depth_refine=None, depth_refine_iter=None, depth_refine_threshold=None,
                 depth_scale=None, vertex_scale=0.001, device="cuda", precision=None, max_batch=64, use_cuda_graph=True):
        """Reference arguments (predictor_gdrn.py:45-50):
          config_file_path   reference-style python config (configs/gdrn/**.py); None -> the YCB-V a6 defaults
          ckpt_file_path     torch checkpoint ({"model": state_dict} or a bare state_dict, "_module." prefixes stripped
                             like MyCheckpointer(prefix_to_remove="_module.")); None -> weights must come via state_dict
          camera_json_path   BOP camera.json (fx, fy, cx, cy, depth_scale)
          path_to_obj_models directory of obj_{id:06d}.ply (millimetres, scaled by vertex_scale = 0.001 like the
                             reference's args.vertex_scale): extents come from the vertex bounding boxes (_get_extents,
                             :478-498) and the meshes feed depth refine
        Keyword-only: the same pieces already loaded (cam 3x3, objs {obj_id: name}, extents {obj_id: (3,)} metres,
        models {obj_id: (verts [V,3] metres, faces [F,3])}, state_dict).

        Per-object models (the reference's configs/gdrn/*SO/**: one class-agnostic network per object): pass
        ckpt_file_path={obj_id: path} or state_dict={obj_id: state_dict}, and config_file_path as one per-object config
        shared by all of them or {obj_id: path}.  inference() then sends every ROI to its object's network
        (PerObjectGDRN); preprocessing and post-processing are unchanged."""
        self.device = torch.device(device)
        # ---- config (predictor_gdrn.py:52-72: eval_only, TEST.USE_PNP=True, TEST.USE_DEPTH_REFINE=False, ...) ----
        obj_cfgs = None
        if isinstance(config_file_path, Mapping):
            obj_cfgs = {int(k): load_py_config(v) for k, v in config_file_path.items()}
            if cfg is None:
                cfg = next(iter(obj_cfgs.values()))   # predictor-level settings (TEST.*, INPUT.*) come from the first
            config_file_path = None
        if cfg is None and config_file_path is not None:
            cfg = load_py_config(config_file_path)
        self.objs_dir = path_to_obj_models
        self.vertex_scale = vertex_scale
        # ---- objects: {obj_id: name}; the reference hard-codes a placeholder dict ("set your trained object names") ----
        if objs is None:
            if path_to_obj_models is None:
                raise ValueError("GdrnPredictor needs objs={obj_id: name} or path_to_obj_models")
            ids = sorted(int(re.search(r"obj_(\d+)\.ply$", p).group(1)) for p in glob.glob(os.path.join(path_to_obj_models, "obj_*.ply")))
            objs = {i: "obj_%06d" % i for i in ids}
        self.objs = dict(objs)
        self.cls_names = list(self.objs.values())
        self.obj_ids = list(self.objs.keys())
        nc = num_classes or _cfg_get(cfg, "MODEL.POSE_NET.NUM_CLASSES", None) or len(self.obj_ids)
        if cfg is None:
            cfg = default_cfg(num_classes=nc)
        self.cfg = cfg
        T = cfg.TEST
        T.USE_PNP = bool(True if use_pnp is None else use_pnp)   # the reference predictor forces TEST.USE_PNP=True (:58)
        T.USE_DEPTH_REFINE = bool(_cfg_get(cfg, "TEST.USE_DEPTH_REFINE", False) if use_depth_refine is None else use_depth_refine)
        T.DEPTH_REFINE_ITER = depth_refine_iter or _cfg_get(cfg, "TEST.DEPTH_REFINE_ITER", 2)
        T.DEPTH_REFINE_THRESHOLD = depth_refine_threshold or _cfg_get(cfg, "TEST.DEPTH_REFINE_THRESHOLD", 0.8)
        self.dzi_pad_scale = float(_cfg_get(cfg, "INPUT.DZI_PAD_SCALE", 1.5))
        self.pixel_mean = tuple(_cfg_get(cfg, "MODEL.PIXEL_MEAN", (0.0, 0.0, 0.0)))
        self.pixel_std = tuple(_cfg_get(cfg, "MODEL.PIXEL_STD", (255.0, 255.0, 255.0)))
        self.mask_thr = float(_cfg_get(cfg, "MODEL.POSE_NET.GEO_HEAD.MASK_THR_TEST", 0.5))
        # ---- camera (predictor_gdrn.py:83-89) ----
        self.depth_scale = 1.0 if depth_scale is None else depth_scale
        if cam is None:
            if camera_json_path is None:
                raise ValueError("GdrnPredictor needs cam=3x3 or camera_json_path")
            with open(camera_json_path) as f:
                cj = json.load(f)
            cam = [[cj["fx"], 0.0, cj["cx"]], [0.0, cj["fy"], cj["cy"]], [0.0, 0.0, 1.0]]
            if depth_scale is None:
                self.depth_scale = cj.get("depth_scale", 1.0)
        self.cam = np.asarray(cam, np.float32)
        # ---- object models / extents (_get_extents, predictor_gdrn.py:478-498; load_models :102-110) ----
        self.obj_models = {}
        if extents is None:
            if path_to_obj_models is None:
                raise ValueError("GdrnPredictor needs extents={obj_id: (3,)} or path_to_obj_models")
            extents, loaded = {}, {}
            for i in self.obj_ids:
                m = load_ply(os.path.join(path_to_obj_models, "obj_%06d.ply" % i), vertex_scale=vertex_scale)
                self.obj_models[i] = m
                pts = m["pts"]
                extents[i] = (pts.max(axis=0) - pts.min(axis=0)).astype(np.float32)
                if "faces" in m:
                    loaded[i] = (pts.astype(np.float32), m["faces"].astype(np.int32))
            if models is None and len(loaded) == len(self.obj_ids):
                models = loaded
        self.extents = {k: np.asarray(v, np.float32) for k, v in extents.items()}
        # ---- model (set_eval_model, predictor_gdrn.py:113-122) ----
        per_object_sd = isinstance(state_dict, Mapping) and bool(state_dict) and all(
            isinstance(v, Mapping) for v in state_dict.values())
        if obj_cfgs is not None or isinstance(ckpt_file_path, Mapping) or per_object_sd:
            self.model = self._per_object_model(obj_cfgs, ckpt_file_path, state_dict if per_object_sd else None,
                                                max_batch, precision, use_cuda_graph)
        else:
            self.model = self._load(GDRN_DoubleMask(self.cfg, arch=_arch(self.cfg), max_batch=max_batch,
                                                    precision=precision), ckpt_file_path, state_dict)
        self.ren_models = None
        if models is not None:
            self.ren_models = [Model3D(*models[i], device=self.device) for i in self.obj_ids]
        # per-image latency path: the per-ROI bookkeeping of one image travels in ONE pinned host block + one H2D copy,
        # the crops are written straight into per-batch-size static buffers, and the ~160 launches of a forward over them
        # are replayed as one CUDA graph (predictor_gdrn.py runs 5-ROI batches: launch-latency bound otherwise)
        self.use_cuda_graph = bool(use_cuda_graph)
        self._coord_grids = {}     # (H, W) -> [H,W,2] normalised coordinate grid on the device
        self._static = {}          # n -> dict of static input tensors (+ pinned staging, + captured graph)

    def _load(self, model, ckpt_file_path, state_dict):
        if state_dict is None and ckpt_file_path is not None:
            ck = torch.load(ckpt_file_path, map_location="cpu")
            state_dict = ck.get("model", ck)
            state_dict = {k[len("_module."):] if k.startswith("_module.") else k: v for k, v in state_dict.items()}
        if state_dict is not None:
            model.load_state_dict(state_dict)
        return model.to(self.device)

    def _per_object_model(self, obj_cfgs, ckpts, state_dicts, max_batch, precision, use_cuda_graph):
        """One class-agnostic GDRN_DoubleMask per object, keyed by the detector label (the index of the object in
        obj_ids, which is what preprocessing() stores in roi_cls)."""
        ckpts = {int(k): v for k, v in (ckpts or {}).items()}
        state_dicts = {int(k): v for k, v in (state_dicts or {}).items()}
        ids = sorted(set(ckpts) | set(state_dicts) or set(obj_cfgs or {}))
        unknown = [i for i in ids if i not in self.objs]
        if unknown:
            raise ValueError(f"per-object weights / configs for obj_id(s) {unknown} that are not in objs {self.obj_ids}")
        T = self.cfg.TEST
        members = {}
        for oid in ids:
            mcfg = (obj_cfgs or {}).get(oid, self.cfg)
            for k in ("USE_PNP", "USE_DEPTH_REFINE", "DEPTH_REFINE_ITER", "DEPTH_REFINE_THRESHOLD"):
                setattr(mcfg.TEST, k, getattr(T, k))   # the predictor's settings apply to every member
            m = GDRN_DoubleMask(mcfg, arch=_arch(mcfg), max_batch=max_batch, precision=precision)
            members[self.obj_ids.index(oid)] = self._load(m, ckpts.get(oid), state_dicts.get(oid))
        return PerObjectGDRN(members, use_cuda_graph=use_cuda_graph)

    # ---- preprocessing (predictor_gdrn.py:301-476) ---------------------------------------------
    def preprocessing(self, outputs, image, depth_img=None):
        """outputs: [n,7] detections (x1,y1,x2,y2,score,cls_score,cls) like the YOLOX stage; image: HxWx3 BGR uint8;
        depth_img: HxW (scaled by depth_scale like the reference).  Per-ROI bookkeeping follows predictor_gdrn.py:396-415
        (centre, bw/bh >= 1, scale = min(max(bw,bh)*DZI_PAD_SCALE, max(H,W)), resize_ratio = out_res/scale); the crops
        -- the reference's per-ROI cv2.warpAffine loop (:417-438) -- are three batched GPU launches with OpenCV's exact
        arithmetic (csrc/crop_resize.cu)."""
        dev = self.device
        det = np.asarray(outputs.detach().cpu() if torch.is_tensor(outputs) else outputs, np.float32).reshape(-1, 7)
        n = det.shape[0]
        image = np.ascontiguousarray(image.detach().cpu().numpy() if torch.is_tensor(image) else image, np.uint8)
        H, W = image.shape[:2]
        in_res, out_res = 256, 64
        st = self._static_buffers(n)
        hf, hd = st["host_f32"], st["host_f64"]      # pinned: [n,18] f32 (centre 2, wh 2, scale, ratio, extent 3, cam 9), [n,12] f64 (M_in, M_out)
        cls_np = det[:, 6].astype(np.int64)
        for i in range(n):
            x1, y1, x2, y2 = det[i, :4]
            c = np.array([0.5 * (x1 + x2), 0.5 * (y1 + y2)])
            bw, bh = max(x2 - x1, 1), max(y2 - y1, 1)
            scale = min(max(bh, bw) * self.dzi_pad_scale, max(H, W)) * 1.0
            hf[i, 0:2] = torch.from_numpy(c.astype(np.float32))
            hf[i, 2], hf[i, 3], hf[i, 4], hf[i, 5] = float(bw), float(bh), float(np.float32(scale)), float(np.float32(out_res / np.float32(scale)))
            hf[i, 6:9] = torch.from_numpy(self.extents[self.obj_ids[int(cls_np[i])]])
            hd[i, 0:6] = torch.from_numpy(get_affine_transform(c, scale, 0, in_res).reshape(6))
            hd[i, 6:12] = torch.from_numpy(get_affine_transform(c, scale, 0, out_res).reshape(6))
        if n:
            hf[:, 9:18] = torch.from_numpy(self.cam.reshape(1, 9))
            st["host_cls"].copy_(torch.from_numpy(cls_np))
        with torch.cuda.device(dev):
            # one small H2D per dtype (pinned, asynchronous), then device-side slices into the static input tensors
            st["dev_f32"].copy_(hf, non_blocking=True)
            st["dev_f64"].copy_(hd, non_blocking=True)
            st["roi_cls"].copy_(st["host_cls"], non_blocking=True)
            df = st["dev_f32"]
            st["roi_center"].copy_(df[:, 0:2]); st["roi_wh"].copy_(df[:, 2:4]); st["scale"].copy_(df[:, 4]); st["resize_ratio"].copy_(df[:, 5])
            st["roi_extent"].copy_(df[:, 6:9]); st["roi_cam"].copy_(df[:, 9:18].reshape(n, 3, 3))
            M_in, M_out = st["dev_f64"][:, 0:6], st["dev_f64"][:, 6:12]
            img_d = torch.from_numpy(image).to(dev, non_blocking=True)
            crop_resize_image(img_d, M_in, in_res, self.pixel_mean, self.pixel_std, out=st["roi_img"])   # PIXEL_MEAN 0 / PIXEL_STD 255
            coord = self._coord_grids.get((H, W))
            if coord is None:
                # get_2d_coord_np(W, H, low=0, high=1) (data_utils.py:304-323): linspace(endpoint=False) grid, [H,W,2] (x, y)
                xs = torch.from_numpy(np.linspace(0, 1, W, endpoint=False, dtype=np.float32))
                ys = torch.from_numpy(np.linspace(0, 1, H, endpoint=False, dtype=np.float32))
                coord = torch.stack([xs[None, :].expand(H, W), ys[:, None].expand(H, W)], dim=2).contiguous().to(dev)
                self._coord_grids[(H, W)] = coord
            crop_resize_float(coord, M_out, out_res, out=st["roi_coord_2d"])
        data = {
            "roi_img": st["roi_img"], "roi_cls": st["roi_cls"], "roi_coord_2d": st["roi_coord_2d"],
            "roi_cam": st["roi_cam"], "cam": st["roi_cam"],
            "roi_center": st["roi_center"], "bbox_center": st["roi_center"], "roi_wh": st["roi_wh"],
            "scale": st["scale"], "resize_ratio": st["resize_ratio"], "roi_extent": st["roi_extent"],
            "im_H": torch.full((n,), H, dtype=torch.float32), "im_W": torch.full((n,), W, dtype=torch.float32),
            "score": torch.from_numpy(det[:, 4] * det[:, 5]), "bbox_est": torch.from_numpy(det[:, :4].copy()),
            "_static_n": n,
        }
        if depth_img is not None:
            with torch.cuda.device(dev):
                d = torch.from_numpy(np.ascontiguousarray(np.asarray(depth_img, np.float32) * np.float32(self.depth_scale))).to(dev)
                data["roi_depth"] = crop_resize_float(d, st["dev_f64"][:, 0:6], in_res, nearest=True)      # [n,1,256,256] like the reference
        return data

    def _static_buffers(self, n):
        """Static device tensors (and their pinned staging) for a batch of n ROIs; allocated once per n.  NOTE: the tensors
        of a returned data_dict are these buffers: they are overwritten by the next preprocessing() of the same batch
        size (the reference allocates fresh tensors per call; clone them to keep a batch alive across calls)."""
        st = self._static.get(n)
        if st is None:
            dev = self.device
            z = lambda *shape, dtype=torch.float32: torch.zeros(shape, dtype=dtype, device=dev)
            st = {
                "host_f32": torch.zeros((n, 18), dtype=torch.float32).pin_memory() if n else torch.zeros((0, 18)),
                "host_f64": torch.zeros((n, 12), dtype=torch.float64).pin_memory() if n else torch.zeros((0, 12), dtype=torch.float64),
                "host_cls": torch.zeros((n,), dtype=torch.int64).pin_memory() if n else torch.zeros((0,), dtype=torch.int64),
                "dev_f32": z(n, 18), "dev_f64": z(n, 12, dtype=torch.float64), "roi_cls": z(n, dtype=torch.int64),
                "roi_img": z(n, 3, 256, 256), "roi_coord_2d": z(n, 2, 64, 64), "roi_cam": z(n, 3, 3), "roi_center": z(n, 2),
                "roi_wh": z(n, 2), "scale": z(n), "resize_ratio": z(n), "roi_extent": z(n, 3), "graph": None,
            }
            self._static[n] = st
        return st

    # ---- inference (predictor_gdrn.py:122-147) --------------------------------------------------
    @torch.no_grad()
    def inference(self, data_dict):
        n = data_dict["roi_img"].shape[0]
        if isinstance(self.model, PerObjectGDRN):   # each ROI to its object's network (graphs per member and size)
            out = self.model(
                data_dict["roi_img"], roi_classes=data_dict["roi_cls"], roi_cams=data_dict["roi_cam"],
                roi_whs=data_dict["roi_wh"], roi_centers=data_dict["roi_center"], resize_ratios=data_dict["resize_ratio"],
                roi_coord_2d=data_dict.get("roi_coord_2d"), roi_extents=data_dict.get("roi_extent"))
            torch.cuda.synchronize(self.device)
            return out
        st = self._static.get(data_dict.get("_static_n", -1))
        graph_ok = (self.use_cuda_graph and st is not None and 1 <= n <= self.model.max_batch
                    and data_dict["roi_img"] is st["roi_img"])       # the batch still lives in the static buffers
        if graph_ok:
            with torch.cuda.device(self.device):
                if st["graph"] is None:
                    st["graph"] = self.model.capture_graph({
                        "roi_img": st["roi_img"], "roi_classes": st["roi_cls"], "roi_coord_2d": st["roi_coord_2d"],
                        "roi_cams": st["roi_cam"], "roi_centers": st["roi_center"], "roi_whs": st["roi_wh"],
                        "roi_extents": st["roi_extent"], "resize_ratios": st["resize_ratio"]})
                replay, out = st["graph"]
                replay()
        else:
            out = self.model(
                data_dict["roi_img"], roi_classes=data_dict["roi_cls"], roi_cams=data_dict["roi_cam"],
                roi_whs=data_dict["roi_wh"], roi_centers=data_dict["roi_center"], resize_ratios=data_dict["resize_ratio"],
                roi_coord_2d=data_dict.get("roi_coord_2d"), roi_extents=data_dict.get("roi_extent"))
        torch.cuda.synchronize(self.device)
        return out

    # ---- postprocessing (predictor_gdrn.py:149-191) ---------------------------------------------
    def postprocessing(self, data_dict, out_dict):
        rot = out_dict["rot"]
        trans = out_dict["trans"]
        n = rot.shape[0]
        if self.cfg.TEST.USE_PNP and n > 0:
            # get_pnp_ransac_pose for every ROI (gdrn_evaluator.py:1122-1221: EPnP RANSAC, reprojErr 3 px, 100 iters),
            # batched on the GPU; ROIs with < 4 correspondences get the reference's -100 sentinel pose
            from .pnp_ransac import pnp_ransac_from_maps

            poses = pnp_ransac_from_maps(out_dict["coor_x"], out_dict["coor_y"], out_dict["coor_z"], out_dict["mask"],
                                         data_dict["roi_coord_2d"], data_dict["im_H"], data_dict["im_W"], data_dict["roi_extent"],
                                         data_dict["cam"], mask_thr=self.mask_thr)
            rot, trans = poses[:, :, :3].contiguous(), poses[:, :, 3].contiguous()
            out_dict = dict(out_dict, rot=rot, trans=trans)
        if self.cfg.TEST.USE_DEPTH_REFINE:
            trans = self.process_depth_refine(data_dict, out_dict)
        R = rot.detach().cpu().numpy()
        t = trans.detach().cpu().numpy()
        data_dict["cur_res"] = []
        poses = {}
        for i in range(n):
            oid = self.obj_ids[int(data_dict["roi_cls"][i])]
            data_dict["cur_res"].append({"obj_id": oid, "score": float(data_dict["score"][i]),
                                         "bbox_est": np.asarray(data_dict["bbox_est"][i]), "R": R[i], "t": t[i]})
            pose = np.eye(4)
            pose[:3, :3], pose[:3, 3] = R[i], t[i]
            poses[self.objs.get(oid)] = pose
        return poses

    # ---- fast depth refine (predictor_gdrn.py:195-286), batched on the GPU ----------------------
    def process_depth_refine(self, inputs, out_dict):
        if self.ren_models is None:
            raise RuntimeError("depth refine needs object meshes (models=... or path_to_obj_models)")
        n = out_dict["rot"].shape[0]
        crop_xy = inputs["roi_center"] - inputs["scale"].view(n, 1) / 2
        K_crop = get_K_crop_resize(inputs["roi_cam"], crop_xy, (64.0 / inputs["scale"]).view(n, 1))
        xyz = torch.cat([out_dict["coor_x"], out_dict["coor_y"], out_dict["coor_z"]], dim=1)
        # depth_sensor_crop = cv2.resize(roi_depth[i].squeeze(), (64, 64)) (predictor_gdrn.py:238): for the exact 4:1
        # ratio INTER_LINEAR samples at 4*d + 1.5, i.e. the mean of the centre 2x2 of every 4x4 cell (weights 1/2, 1/2 per
        # axis).  Computed as ((a+b)+(c+d))/4 = the correctly rounded mean; cv2's two-pass float path differs from it by
        # at most 1 ulp on ~8 % of the pixels (double rounding), far below the sensor noise the refinement thresholds on
        d = inputs["roi_depth"]
        if d.dim() == 4:
            d = d[:, 0]
        if d.shape[-1] == 256:
            d = ((d[:, 1::4, 1::4] + d[:, 1::4, 2::4]) + (d[:, 2::4, 1::4] + d[:, 2::4, 2::4])) * 0.25
        return depth_refine([m.vertices for m in self.ren_models], [m.faces for m in self.ren_models], out_dict["rot"],
                            out_dict["trans"], K_crop, xyz, out_dict["mask"], d.contiguous(),
                            iters=self.cfg.TEST.DEPTH_REFINE_ITER, thresh=self.cfg.TEST.DEPTH_REFINE_THRESHOLD,
                            mesh_ids=inputs["roi_cls"])


def _arch(cfg):
    return str(_cfg_get(cfg, "MODEL.POSE_NET.BACKBONE.INIT_CFG.type", "timm/convnext_base")).split("/")[-1]
