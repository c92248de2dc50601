"""YoloPredictor -- the detector stage of the reference demo (core/gdrn_modeling/demo/predictor_yolo.py), on the YOLOX
network of yolox_model.py and the keep-single-instance post-process of csrc/yolox_net.cu.

``YoloPredictor(exp_name, config_file_path, ckpt_file_path, fuse, fp16).inference(image)`` returns what the reference
returns: a list with one [n, 7] tensor (x1, y1, x2, y2, obj_conf, class_conf, class) on the device, or ``[None]``, and
that list goes into ``GdrnPredictor.preprocessing(outputs=...)`` unchanged.

Deliberate differences from the reference:
  (a) classes without a detection are left out; the reference fills their rows with torch.rand values
      (predictor_yolo.py:108) that then take part in the NMS and come out as detections;
  (b) boxes are divided by the letterbox ratio r, so they are in the coordinates of the image passed in.  The reference
      discards r (:150): its boxes are right only when r = 1, which holds for 640x480 images such as LM-O and YCB-V
      with the shipped 640x640 test size, and for those images the results are the same.
"""
import numpy as np
import torch

from . import _lib
from .yolox_model import YOLOX, load_yolox_config, tta_scales


def preproc(img, input_size):
    """det/yolox/data/data_augment.py:161-177 (ValTransform(legacy=False)): letterbox into input_size (h, w) with
    pad 114, cv2 INTER_LINEAR, BGR kept, no normalisation -> ([3, h, w] float32, r)."""
    import cv2

    if img.ndim == 3:
        padded = np.ones((input_size[0], input_size[1], 3), dtype=np.uint8) * 114
    else:
        padded = np.ones(input_size, dtype=np.uint8) * 114
    r = min(input_size[0] / img.shape[0], input_size[1] / img.shape[1])
    resized = cv2.resize(img, (int(img.shape[1] * r), int(img.shape[0] * r)), interpolation=cv2.INTER_LINEAR).astype(np.uint8)
    padded[: int(img.shape[0] * r), : int(img.shape[1] * r)] = resized
    return np.ascontiguousarray(padded.transpose(2, 0, 1), dtype=np.float32), r


@_lib.on_device(0)
def postprocess_single_instance(det_preds, num_classes, conf_thre, nms_thre, workspace=None):
    """YoloPredictor.postprocess(class_agnostic=True, keep_single_instance=True) (predictor_yolo.py:84-140) on the
    device: per class the highest-scoring anchor with obj * class_conf >= conf_thre (the first one on ties), then
    class-agnostic NMS as torchvision's CPU nms decides it (IoU compared with nms_thre as a double), rows sorted by
    class.  -> (dets [B, nc, 7], n_det [B] int32), no synchronisation.  ``workspace``: a one-element list that holds
    the workspace across calls (grown when a call needs more)."""
    if not det_preds.is_cuda:
        raise _lib.GdrnError("keep-single-instance post-process needs CUDA tensors (no CPU fallback)")
    B, A, C = det_preds.shape
    if C != 5 + num_classes:
        raise ValueError(f"det_preds has {C} columns, expected 5 + {num_classes}")
    p = det_preds.detach().to(torch.float32).contiguous()
    dets = torch.zeros((B, num_classes, 7), dtype=torch.float32, device=p.device)
    n_det = torch.zeros((B,), dtype=torch.int32, device=p.device)
    L = _lib.lib()
    nb = L.yolox_postprocess_single_workspace_bytes(B, A, num_classes)
    if workspace is None:
        ws = torch.empty(nb, dtype=torch.uint8, device=p.device)
    else:
        if workspace[0] is None or workspace[0].numel() < nb or workspace[0].device != p.device:
            workspace[0] = torch.empty(nb, dtype=torch.uint8, device=p.device)
        ws = workspace[0]
    _lib.check(L.yolox_postprocess_single(_lib.ptr(p), B, A, int(num_classes), float(conf_thre), float(nms_thre),
                                          _lib.ptr(dets), _lib.ptr(n_det), _lib.ptr(ws), ws.numel(), _lib.current_stream()),
               "yolox_postprocess_single")
    return dets, n_det


class YoloPredictor:
    def __init__(self, exp_name="yolox-x", config_file_path=None, ckpt_file_path=None, fuse=True, fp16=False, *,
                 state_dict=None, precision=None, device="cuda", cfg=None, max_batch=1, use_cuda_graph=True, augment=False):
        """Reference arguments (predictor_yolo.py:29-34).  ``exp_name`` is accepted and unused: the config file names
        the model.  ``fuse`` is accepted: the BatchNorms are always folded.  ``fp16=True`` selects the bf16 mode (the
        nearest here to the reference's half regime); an explicit ``precision`` wins.  Keyword-only: ``state_dict``
        instead of a checkpoint, ``cfg`` (the namespace load_yolox_config returns) instead of a config file, and
        ``augment=True`` to run the multi-scale test-time augmentation over ``cfg.scales`` (the reference predictor
        never passes augment, hence the default)."""
        self.exp_name, self.fuse, self.augment = exp_name, fuse, bool(augment)
        if cfg is None:
            if config_file_path is None:
                raise ValueError("YoloPredictor needs config_file_path or cfg=")
            cfg = load_yolox_config(config_file_path)
        self.cfg = cfg
        self.device = torch.device(device)
        self.precision = precision or ("bf16" if fp16 else "bf16x3")
        self.model = YOLOX(cfg.depth, cfg.width, cfg.num_classes, max_batch=max_batch, precision=self.precision).eval()
        if state_dict is None:
            if ckpt_file_path is None:
                raise ValueError("YoloPredictor needs ckpt_file_path or state_dict=")
            ck = torch.load(ckpt_file_path, map_location="cpu")
            state_dict = ck.get("model", ck)
        state_dict = {k[len("_module."):] if k.startswith("_module.") else k: v for k, v in state_dict.items()}
        self.model.load_state_dict(state_dict)
        self.model.to(self.device)
        self.use_cuda_graph = bool(use_cuda_graph)
        self._graph = None   # (replay, static input, static det_preds, scales)

    def _forward(self, img):
        kw = {"augment": True, "cfg": self.cfg} if self.augment else {}
        if not self.use_cuda_graph:
            return self.model(img, **kw)["det_preds"]
        scales = tta_scales(self.cfg) if self.augment else None
        if self._graph is None or self._graph[1].shape != img.shape or self._graph[3] != scales:
            static = img.clone()
            replay, out = self.model.capture_graph(static, **kw)
            self._graph = (replay, static, out["det_preds"], scales)
        replay, static, det, _ = self._graph
        static.copy_(img)
        replay()
        return det

    def inference(self, image):
        """image: HxWx3 BGR uint8 -> [dets [n, 7] CUDA tensor] or [None] (predictor_yolo.py:142-171)."""
        image = image.detach().cpu().numpy() if torch.is_tensor(image) else np.asarray(image)
        img, r = preproc(image, self.cfg.test_size)
        with torch.cuda.device(self.device):
            x = torch.from_numpy(img).unsqueeze(0).to(self.device)
            det_preds = self._forward(x)
            dets, n_det = postprocess_single_instance(det_preds, self.cfg.num_classes, self.cfg.conf_thr, self.cfg.nms_thr)
            n = int(n_det[0].item())
            if n == 0:
                return [None]
            out = dets[0, :n].clone()
            out[:, :4] /= r
        return [out]
