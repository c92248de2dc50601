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


# ---------------------------------------------------------------------------------------------------------------------
# the engine's layer plan, one step at a time (yolox_model_step_info / yolox_model_run_step): the folded and merged
# weights of every packed conv, restated from the reference's modules, and one torch op per step kind
# ---------------------------------------------------------------------------------------------------------------------
def fold(sd, prefix):
    """(w [Cout, Cin, k, k], b [Cout]) float64 of one BaseConv with its BatchNorm folded in (fuse_conv_and_bn,
    det/yolox/utils/model_utils.py:33-58, eps 1e-3), from an unfused (conv + bn) or a fused (conv bias) state dict."""
    w = sd[prefix + ".conv.weight"].double()
    cb = sd.get(prefix + ".conv.bias")
    cb = torch.zeros(w.shape[0], dtype=torch.float64, device=w.device) if cb is None else cb.double()
    if prefix + ".bn.weight" not in sd:
        return w, cb
    g, beta = sd[prefix + ".bn.weight"].double(), sd[prefix + ".bn.bias"].double()
    mean, var = sd[prefix + ".bn.running_mean"].double(), sd[prefix + ".bn.running_var"].double()
    s = g / torch.sqrt(var + BN_EPS)
    return w * s[:, None, None, None], s * cb + (beta - g * mean / torch.sqrt(var + BN_EPS))


def packed_conv(sd, name):
    """(w, b) float64 of one conv of the engine's step table by its packed name: a BaseConv prefix folded; the merged head
    convs head.conv0.k = [cls_convs.k.0 | reg_convs.k.0] and head.regobj.k = [reg_preds.k | obj_preds.k] along N;
    head.cls.k = cls_preds.k; the stem's 12 Focus input channels padded to 16 with zero weights."""
    level = name.rsplit(".", 1)[-1]
    pred = lambda p: (sd[p + ".weight"].double(), sd[p + ".bias"].double())  # noqa: E731
    if name.startswith("head.conv0."):
        parts = [fold(sd, f"head.cls_convs.{level}.0"), fold(sd, f"head.reg_convs.{level}.0")]
    elif name.startswith("head.regobj."):
        parts = [pred(f"head.reg_preds.{level}"), pred(f"head.obj_preds.{level}")]
    elif name.startswith("head.cls."):
        parts = [pred(f"head.cls_preds.{level}")]
    else:
        parts = [fold(sd, name)]
    w, b = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    if name.endswith("stem.conv"):
        w = F.pad(w, (0, 0, 0, 0, 0, 16 - w.shape[1]))
    return w, b


def conv_op(x, w, b, stride, act, resid=None):
    """x [B, Cin, h, w] -> act(conv(x) + b) (+ resid): the engine's conv epilogue adds the shortcut after SiLU."""
    y = F.conv2d(x, w, b, stride=stride, padding=(w.shape[-1] - 1) // 2)
    if act:
        y = y * torch.sigmoid(y)
    return y if resid is None else y + resid


def focus_op(x):
    """[B, 3, H, W] -> [B, 16, H/2, W/2]: Focus's space-to-depth (TL, BL, TR, BR) x 3, then 4 zero channels."""
    y = torch.cat((x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]), 1)
    return F.pad(y, (0, 0, 0, 0, 0, 4))


def spp_op(x):
    """[B, C, h, w] -> [B, 3C, h, w]: the 5 / 9 / 13 max-pools of SPPBottleneck (stride 1, -inf padding)."""
    return torch.cat([F.max_pool2d(x, k, 1, k // 2) for k in (5, 9, 13)], 1)


def upsample_op(x):
    return F.interpolate(x, scale_factor=2, mode="nearest")


def head_op(raw, stride, inv_scale=1.0):
    """raw [B, 5 + nc, h, w] (reg 4 | obj | cls) -> [B, h*w, 5 + nc] decoded as YOLOXHead.decode_outputs:
    (xy + grid) * stride, exp(wh) * stride, sigmoid(obj), sigmoid(cls); then the box columns times inv_scale (the
    test-time-augmentation de-scale, 1 for the plain forward).  In the dtype of raw: float32 restates the kernel's
    round-to-nearest ops one for one."""
    B, C, h, w = raw.shape
    o = raw.flatten(2).permute(0, 2, 1)
    yv, xv = torch.meshgrid(torch.arange(h, device=raw.device), torch.arange(w, device=raw.device), indexing="ij")
    grid = torch.stack((xv, yv), 2).view(1, -1, 2).to(o)
    box = torch.cat([(o[..., :2] + grid) * stride, torch.exp(o[..., 2:4]) * stride], -1)
    if inv_scale != 1.0:
        box = box * inv_scale
    return torch.cat([box, torch.sigmoid(o[..., 4:])], -1)


def nchw(buf, off, c, h, w):
    """Channel slice [off, off + c) of an engine buffer [B, h*w, ld] as [B, c, h, w]."""
    return buf[:, :, off:off + c].reshape(buf.shape[0], h, w, c).permute(0, 3, 1, 2)


def store(buf, off, y):
    """Write y [B, c, h, w] into channel slice [off, off + c) of an engine buffer [B, h*w, ld]."""
    buf[:, :, off:off + y.shape[1]] = y.permute(0, 2, 3, 1).reshape(buf.shape[0], -1, y.shape[1])


def replay_step(step, bufs, x, det, weights, scale=1.0, a_base=0):
    """Run one step of the engine's step table (a dict with the slots of yolox_model_step_info) on torch buffers
    ``bufs`` ([B, pix, ld] each, any dtype), the input x [B, 3, H, W] and det [B, A_row, 5 + nc]: one torch op per step
    kind.  ``weights``: packed name -> (w, b); ``scale``: the plan's test-time-augmentation scale (1 for plan 0);
    ``a_base``: the plan's anchor base."""
    k = step["kind"]
    if k == "conv":
        w, b = weights[step["name"]]
        inp = nchw(bufs[step["src"]], step["s_off"], step["s_c"], step["in_h"], step["in_w"])
        res = None
        if step["res"] >= 0:
            res = nchw(bufs[step["res"]], step["r_off"], step["d_c"], step["out_h"], step["out_w"])
        y = conv_op(inp, w.to(inp), b.to(inp), step["stride"], step["act"], res)
        store(bufs[step["dst"]], step["d_off"], y)
    elif k == "focus":
        from .yolox_tta_oracle import tta_scale_input

        store(bufs[step["dst"]], 0, focus_op(tta_scale_input(x, scale).to(bufs[step["dst"]])))
    elif k == "spp":
        store(bufs[step["dst"]], step["d_off"], spp_op(nchw(bufs[step["src"]], 0, step["s_c"], step["in_h"], step["in_w"])))
    elif k == "upsample":
        store(bufs[step["dst"]], step["d_off"],
              upsample_op(nchw(bufs[step["src"]], step["s_off"], step["s_c"], step["in_h"], step["in_w"])))
    else:
        raw = nchw(bufs[step["src"]], 0, step["s_c"], step["in_h"], step["in_w"])
        a0 = a_base + step["anchor_off"]
        det[:, a0:a0 + step["in_h"] * step["in_w"]] = head_op(raw, step["level_stride"], 1.0 / scale).to(det)
