"""YOLOX detection post-processing on the GPU (SURVEY.md §8f rank 4): the stage that feeds GdrnPredictor.preprocessing.

Mirrors ``postprocess(det_preds, num_classes, conf_thre, nms_thre, class_agnostic)`` (det/yolox/utils/boxes.py:34-80) and
``YOLOXHead.decode_outputs`` (det/yolox/models/yolo_head.py:239-255) with one call of libgdrn_b200.so per batch
(csrc/yolox_post.cu): decode, filter, class-aware NMS, rows ``(x1, y1, x2, y2, obj_conf, class_conf, class_pred)`` in
descending score order.  The YOLOX network itself is yolox_model.py.  No CPU fallback.
"""
import torch

from . import _lib


@_lib.on_device(0)
def postprocess_padded(det_preds, num_classes, conf_thre=0.7, nms_thre=0.45, class_agnostic=False, hw=None, strides=None,
                       max_out=None, workspace=None):
    """-> (dets [B, max_out, 7], n_det [B] int32), both on the device, no synchronisation.  ``hw`` (list of (rows, cols)
    per pyramid level) + ``strides``: det_preds are RAW head outputs and are decoded here; otherwise they are decoded
    (cx, cy, w, h) boxes, as YOLOXHead returns them with decode_in_inference.  ``workspace``: a one-element list that
    holds the NMS workspace across calls (grown when a call needs more), so a loop does not allocate it per batch."""
    if not det_preds.is_cuda:
        raise _lib.GdrnError("yolox postprocess needs CUDA tensors (no CPU fallback)")
    dev = det_preds.device
    B, A, C = det_preds.shape
    assert C == 5 + num_classes, (C, num_classes)
    p = det_preds.detach().to(dtype=torch.float32).contiguous()
    max_out = int(max_out or A)
    dets = torch.zeros((B, max_out, 7), dtype=torch.float32, device=dev)
    n_det = torch.zeros((B,), dtype=torch.int32, device=dev)
    hw_t = st_t = None
    n_levels = 0
    if hw is not None:
        n_levels = len(hw)
        assert strides is not None and len(strides) == n_levels and sum(h * w for h, w in hw) == A
        hw_t = torch.tensor([[int(h), int(w)] for h, w in hw], dtype=torch.int32, device=dev)
        st_t = torch.tensor([int(s) for s in strides], dtype=torch.int32, device=dev)
    L = _lib.lib()
    nb = L.yolox_postprocess_workspace_bytes(B, A)
    if workspace is None:
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    else:
        if workspace[0] is None or workspace[0].numel() < nb or workspace[0].device != dev:
            workspace[0] = torch.empty(nb, dtype=torch.uint8, device=dev)
        ws = workspace[0]
    _lib.check(L.yolox_postprocess(_lib.ptr(p), B, A, int(num_classes), _lib.ptr(hw_t), _lib.ptr(st_t), n_levels, float(conf_thre),
                                   float(nms_thre), int(bool(class_agnostic)), max_out, _lib.ptr(dets), _lib.ptr(n_det), _lib.ptr(ws),
                                   ws.numel(), _lib.current_stream()), "yolox_postprocess")
    return dets, n_det


def postprocess(det_preds, num_classes, conf_thre=0.7, nms_thre=0.45, class_agnostic=False, hw=None, strides=None):
    """Reference signature and return value (det/yolox/utils/boxes.py:34): a list with one [n_i, 7] tensor per image, or
    ``None`` for an image without detections.  The variable-length list needs the counts on the host: ONE device -> host
    copy for the whole batch (the reference synchronises several times per image)."""
    dets, n_det = postprocess_padded(det_preds, num_classes, conf_thre, nms_thre, class_agnostic, hw, strides)
    counts = n_det.cpu().tolist()
    return [dets[i, :c] if c > 0 else None for i, c in enumerate(counts)]
