"""Functional torch restatement of the YOLOX inference forward (det/yolox/models: CSPDarknet, YOLOPAFPN, YOLOXHead with
decode_in_inference) from a state dict with the reference's keys.  Runs in the dtype and on the device of the input
(float64 on the CPU or the GPU for the checks).  Accepts unfused state dicts (conv + BatchNorm, eps 1e-3 as
YOLOX.init_yolo sets it) and fused ones (conv bias, no bn, as fuse_model saves them).

``on_conv(prefix, y)`` (optional) is called with every BaseConv's convolution output before its BatchNorm; it may
write that BatchNorm's running statistics into the state dict (synthetic weights calibrate themselves that way).
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-3


def _t(sd, key, like):
    return sd[key].to(device=like.device, dtype=like.dtype)


def base_conv(sd, prefix, x, stride=1, act=True, on_conv=None):
    w = _t(sd, prefix + ".conv.weight", x)
    k = w.shape[-1]
    bias = _t(sd, prefix + ".conv.bias", x) if prefix + ".conv.bias" in sd else None
    y = F.conv2d(x, w, bias, stride=stride, padding=(k - 1) // 2)
    if prefix + ".bn.weight" in sd:
        if on_conv is not None:
            on_conv(prefix, y)
        mean, var = _t(sd, prefix + ".bn.running_mean", x), _t(sd, prefix + ".bn.running_var", x)
        g, b = _t(sd, prefix + ".bn.weight", x), _t(sd, prefix + ".bn.bias", x)
        y = (y - mean[:, None, None]) / torch.sqrt(var + BN_EPS)[:, None, None] * g[:, None, None] + b[:, None, None]
    return y * torch.sigmoid(y) if act else y


def csp_layer(sd, prefix, x, n, shortcut, on_conv=None):
    x1 = base_conv(sd, prefix + ".conv1", x, on_conv=on_conv)
    x2 = base_conv(sd, prefix + ".conv2", x, on_conv=on_conv)
    for i in range(n):
        y = base_conv(sd, f"{prefix}.m.{i}.conv1", x1, on_conv=on_conv)
        y = base_conv(sd, f"{prefix}.m.{i}.conv2", y, on_conv=on_conv)
        x1 = y + x1 if shortcut else y
    return base_conv(sd, prefix + ".conv3", torch.cat([x1, x2], 1), on_conv=on_conv)


def spp(sd, prefix, x, on_conv=None):
    x = base_conv(sd, prefix + ".conv1", x, on_conv=on_conv)
    x = torch.cat([x] + [F.max_pool2d(x, k, 1, k // 2) for k in (5, 9, 13)], 1)
    return base_conv(sd, prefix + ".conv2", x, on_conv=on_conv)


def yolox_forward(sd, x, depth, num_classes, on_conv=None, strides=(8, 16, 32)):
    """x [B,3,H,W] (BGR, 0..255) -> det_preds [B, A, 5 + num_classes] (decoded boxes, sigmoid scores)."""
    oc = on_conv
    bd = max(round(depth * 3), 1)
    n_fpn = round(3 * depth)
    p = "backbone.backbone."
    x = torch.cat((x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]), 1)
    x = base_conv(sd, p + "stem.conv", x, on_conv=oc)
    x = csp_layer(sd, p + "dark2.1", base_conv(sd, p + "dark2.0", x, 2, on_conv=oc), bd, True, oc)
    d3 = csp_layer(sd, p + "dark3.1", base_conv(sd, p + "dark3.0", x, 2, on_conv=oc), 3 * bd, True, oc)
    d4 = csp_layer(sd, p + "dark4.1", base_conv(sd, p + "dark4.0", d3, 2, on_conv=oc), 3 * bd, True, oc)
    x = spp(sd, p + "dark5.1", base_conv(sd, p + "dark5.0", d4, 2, on_conv=oc), oc)
    d5 = csp_layer(sd, p + "dark5.2", x, bd, False, oc)
    p = "backbone."
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")  # noqa: E731
    fpn_out0 = base_conv(sd, p + "lateral_conv0", d5, on_conv=oc)
    f_out0 = csp_layer(sd, p + "C3_p4", torch.cat([up(fpn_out0), d4], 1), n_fpn, False, oc)
    fpn_out1 = base_conv(sd, p + "reduce_conv1", f_out0, on_conv=oc)
    pan_out2 = csp_layer(sd, p + "C3_p3", torch.cat([up(fpn_out1), d3], 1), n_fpn, False, oc)
    p_out1 = base_conv(sd, p + "bu_conv2", pan_out2, 2, on_conv=oc)
    pan_out1 = csp_layer(sd, p + "C3_n3", torch.cat([p_out1, fpn_out1], 1), n_fpn, False, oc)
    p_out0 = base_conv(sd, p + "bu_conv1", pan_out1, 2, on_conv=oc)
    pan_out0 = csp_layer(sd, p + "C3_n4", torch.cat([p_out0, fpn_out0], 1), n_fpn, False, oc)
    outs = []
    for k, (f, st) in enumerate(zip((pan_out2, pan_out1, pan_out0), strides)):
        h = "head."
        f = base_conv(sd, f"{h}stems.{k}", f, on_conv=oc)
        c = base_conv(sd, f"{h}cls_convs.{k}.1", base_conv(sd, f"{h}cls_convs.{k}.0", f, on_conv=oc), on_conv=oc)
        r = base_conv(sd, f"{h}reg_convs.{k}.1", base_conv(sd, f"{h}reg_convs.{k}.0", f, on_conv=oc), on_conv=oc)
        cls = F.conv2d(c, _t(sd, f"{h}cls_preds.{k}.weight", c), _t(sd, f"{h}cls_preds.{k}.bias", c))
        reg = F.conv2d(r, _t(sd, f"{h}reg_preds.{k}.weight", r), _t(sd, f"{h}reg_preds.{k}.bias", r))
        obj = F.conv2d(r, _t(sd, f"{h}obj_preds.{k}.weight", r), _t(sd, f"{h}obj_preds.{k}.bias", r))
        o = torch.cat([reg, obj.sigmoid(), cls.sigmoid()], 1)
        B, C, hh, ww = o.shape
        o = o.flatten(2).permute(0, 2, 1)
        yv, xv = torch.meshgrid(torch.arange(hh), torch.arange(ww), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, -1, 2).to(o)
        o = torch.cat([(o[..., :2] + grid) * st, torch.exp(o[..., 2:4]) * st, o[..., 4:]], -1)
        outs.append(o)
    return torch.cat(outs, 1)


def keep_single_instance(det, num_classes, conf_thre, nms_thre, ious=None):
    """Host restatement of YoloPredictor.postprocess(class_agnostic=True, keep_single_instance=True) for ONE image's
    decoded det_preds [A, 5 + nc] (predictor_yolo.py:84-140), with classes without a detection dropped instead of
    filled with random rows.  -> [n, 7] float64 numpy array, rows in ascending class order (or None).  ``ious``
    (a list) collects every IoU the NMS compares against its threshold."""
    import numpy as np

    d = np.asarray(det, np.float64)
    box = np.stack([d[:, 0] - d[:, 2] / 2, d[:, 1] - d[:, 3] / 2, d[:, 0] + d[:, 2] / 2, d[:, 1] + d[:, 3] / 2], 1)
    cls_s = d[:, 5:5 + num_classes]
    cc, cp = cls_s.max(1), cls_s.argmax(1)
    score = d[:, 4] * cc
    keep = score >= conf_thre
    rows = np.concatenate([box, d[:, 4:5], cc[:, None], cp[:, None].astype(np.float64)], 1)[keep]
    sc = score[keep]
    sel = []
    for c in range(num_classes):
        idx = np.nonzero(rows[:, 6] == c)[0]
        best, bi = 0.0, -1
        for i in idx:
            if sc[i] > best:
                best, bi = sc[i], i
        if bi >= 0:
            sel.append(bi)
    if not sel:
        return None
    r, s = rows[sel], sc[sel]
    order = sorted(range(len(sel)), key=lambda i: (-s[i], r[i, 6]))
    kept = []
    for i in order:
        ok = True
        for j in kept:
            a, b = r[i], r[j]
            iw = max(min(a[2], b[2]) - max(a[0], b[0]), 0.0)
            ih = max(min(a[3], b[3]) - max(a[1], b[1]), 0.0)
            inter = iw * ih
            iou = inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)
            if ious is not None:
                ious.append(iou)
            if iou > nms_thre:
                ok = False
                break
        if ok:
            kept.append(i)
    out = r[sorted(kept, key=lambda i: r[i, 6])]
    return out
