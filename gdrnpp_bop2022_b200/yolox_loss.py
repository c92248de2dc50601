"""YOLOX training loss on the GPU (DESIGN.md §7q): ``YOLOXHead.get_losses`` (det/yolox/models/yolo_head.py:256-426) as
one set of launches of libgdrn_b200.so per batch (csrc/yolox_loss.cu): SimOTA assignment for every image and GT at
once, the IoU, objectness, class and L1 terms, and their gradients through autograd.  No CPU fallback.

``get_losses`` has the reference method's signature with ``self`` renamed to ``head``, so
``YOLOXHead.get_losses = yolox_loss.get_losses`` swaps it into the reference's own training model.  Differences from the
reference, all deliberate:
  - ``out_dict["num_fg"]`` (num_fg / num_gt) is a 0-d device tensor rather than a Python float, so nothing waits for
    the device;
  - everything is computed in fp32 whatever the dtype of ``outputs``; under AMP (fp16 outputs and labels) this is more
    accurate than the reference, whose IoU loss and candidate test run in fp16.  The losses are fp32 tensors and the
    gradients come back in the input dtype;
  - an image whose GTs have no candidate anchor at all takes no anchors (the reference fails there);
  - equal costs in a GT's k cheapest anchors go to the lower anchor index (torch.topk leaves that order open).
"""
import torch

from . import _lib

_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
_RESULT = 15   # yolox_loss_layout index of result [8] f32
LAYOUT_NAMES = ("nlabel", "cand", "cls_sum", "count", "chooser", "n_cand", "k", "iou_sum", "chosen", "fg", "matched",
                "iou_t", "partial", "partial_fg", "err", "result")


def workspace_layout(B, A, M):
    """(total bytes, {name: byte offset from the 256-aligned workspace base}) of a call's workspace."""
    L = _lib.lib()
    offs = (_lib.c_size_t * len(LAYOUT_NAMES))()
    _lib.check(L.yolox_loss_layout(B, A, M, offs), "yolox_loss_layout")
    return L.yolox_loss_workspace_bytes(B, A, M), dict(zip(LAYOUT_NAMES, offs))


def workspace_view(ws, offsets, name, dtype, shape):
    """A stage result the forward left in its workspace, as a tensor view."""
    base = (-ws.data_ptr()) % 256
    n = 1
    for s in shape:
        n *= s
    nbytes = n * torch.empty((), dtype=dtype).element_size()
    o = base + offsets[name]
    return ws[o:o + nbytes].view(dtype).view(*shape)


def forward_raw(outputs, origin_preds, labels, shifts, num_classes, use_l1, trace=None):
    """One forward call.  outputs [B, A, 5+C] and origin_preds [B, A, 4] (or None) of one dtype, contiguous; labels
    [B, M, 5] f32; shifts [3, A] f32.  -> (workspace, offsets).  ``trace`` (None or zeroed [B, M, A, 3] f32) receives
    (IoU, unpenalised cost, cost) of every candidate pair."""
    B, A, D = outputs.shape
    M = labels.shape[1]
    if D != 5 + num_classes:
        raise ValueError(f"outputs has {D} channels, expected 5 + num_classes = {5 + num_classes}")
    nb, offs = workspace_layout(B, A, M)
    ws = torch.empty(nb, dtype=torch.uint8, device=outputs.device)
    _lib.check(_lib.lib().yolox_loss_forward(
        _lib.ptr(outputs), _lib.ptr(origin_preds), _DTYPES[outputs.dtype], _lib.ptr(labels), _lib.ptr(shifts), B, A,
        num_classes, M, int(use_l1), _lib.ptr(trace), _lib.ptr(ws), ws.numel(), _lib.current_stream()),
        "yolox_loss_forward")
    return ws, offs


class _YoloxLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, outputs, origin_preds, labels, shifts, num_classes, use_l1):
        ws, offs = forward_raw(outputs, origin_preds, labels, shifts, num_classes, use_l1)
        res = workspace_view(ws, offs, "result", torch.float32, (8,))
        # F.one_hot rejects a class id outside [0, C): one flag read back per call
        if res[6].item() != 0:
            raise ValueError(f"labels hold a class id outside [0, num_classes={num_classes})")
        ctx.save_for_backward(outputs, origin_preds, labels, shifts, ws)
        ctx.num_classes, ctx.use_l1 = num_classes, use_l1
        ratio = res[5].clone()
        ctx.mark_non_differentiable(ratio)
        return res[:4].clone(), ratio

    @staticmethod
    def backward(ctx, grad_losses, _grad_ratio):
        outputs, origin_preds, labels, shifts, ws = ctx.saved_tensors
        B, A, _ = outputs.shape
        g = grad_losses.to(torch.float32).contiguous()
        grad_out = torch.empty_like(outputs)
        grad_org = torch.empty_like(origin_preds) if ctx.use_l1 else None
        _lib.check(_lib.lib().yolox_loss_backward(
            _lib.ptr(outputs), _lib.ptr(origin_preds), _DTYPES[outputs.dtype], _lib.ptr(labels), _lib.ptr(shifts), B, A,
            ctx.num_classes, labels.shape[1], int(ctx.use_l1), _lib.ptr(g), _lib.ptr(ws), ws.numel(), _lib.ptr(grad_out),
            _lib.ptr(grad_org), _lib.current_stream()), "yolox_loss_backward")
        return grad_out, grad_org, None, None, None, None


def check_head(head):
    """The loss options this implementation covers; anything else is rejected by name."""
    if head.iou_loss.loss_type != "iou":
        raise NotImplementedError(f"iou_loss_type={head.iou_loss.loss_type!r} is not supported (only 'iou')")
    if head.cls_loss_type != "bce":
        raise NotImplementedError(f"cls_loss_type={head.cls_loss_type!r} is not supported (only 'bce')")
    if head.obj_loss_type != "bce":
        raise NotImplementedError(f"obj_loss_type={head.obj_loss_type!r} is not supported (only 'bce')")


def get_losses(head, imgs, x_shifts, y_shifts, expanded_strides, labels, outputs, origin_preds, dtype):
    """YOLOXHead.get_losses on the GPU.  -> (out_dict, loss_dict) with the reference's keys: loss_iou (already times
    reg_weight = 5), loss_conf, loss_cls, loss_l1 (the float 0.0 when head.use_l1 is off); out_dict["num_fg"] =
    num_fg / max(num_gt, 1) as a 0-d device tensor.  ``imgs`` and ``dtype`` are not used."""
    check_head(head)
    if not outputs.is_cuda:
        raise _lib.GdrnError("yolox get_losses needs CUDA tensors (no CPU fallback)")
    if outputs.dtype not in _DTYPES:
        raise TypeError(f"outputs must be float32, float16 or bfloat16, got {outputs.dtype}")
    use_l1 = bool(head.use_l1)
    with torch.cuda.device(outputs.device):
        out = outputs.contiguous()
        org = torch.cat(origin_preds, 1).to(out.dtype).contiguous() if use_l1 else None
        shifts = torch.cat(list(x_shifts) + list(y_shifts) + list(expanded_strides), 1).to(
            device=out.device, dtype=torch.float32).reshape(3, -1)
        if shifts.shape[1] != out.shape[1]:
            raise ValueError(f"x_shifts / y_shifts / expanded_strides cover {shifts.shape[1]} anchors, outputs has "
                             f"{out.shape[1]}")
        lab = labels.to(device=out.device, dtype=torch.float32).contiguous()
        losses, ratio = _YoloxLoss.apply(out, org, lab, shifts, int(head.num_classes), use_l1)
    loss_iou, loss_obj, loss_cls, loss_l1 = losses.unbind(0)
    loss_dict = {"loss_iou": loss_iou, "loss_conf": loss_obj, "loss_l1": loss_l1 if use_l1 else 0.0,
                 "loss_cls": loss_cls}
    return {"num_fg": ratio}, loss_dict
