"""Functional torch restatement of YOLOX's multi-scale test-time augmentation (YOLOX.forward(augment=True, cfg),
det/yolox/models/yolox.py:53-86, with the scaled input of model_utils.scale_img) on top of the network forward of
yolox_oracle.py.  Per scale s: the input resized bilinearly (align_corners=False) to int(H*s) x int(W*s) in float32, as
the reference's fp32 test input is, padded on the right and bottom with 0.447 * 255 up to ceil(H*s/32)*32 x
ceil(W*s/32)*32; the network in the dtype of the input; the boxes divided by s; the scales concatenated along the anchor
axis in scale order.
"""
import math

import torch
import torch.nn.functional as F

from .yolox_oracle import yolox_forward

TTA_PAD = 0.447 * 255   # the padding value of the scaled test input (ImageNet mean)


def tta_sizes(h, w, s, gs=32):
    """Sizes of the scaled test input of an h x w input at scale s -> ((content h, w), (padded h, w))."""
    return (int(h * s), int(w * s)), (math.ceil(h * s / gs) * gs, math.ceil(w * s / gs) * gs)


def tta_scale_input(x, s, gs=32):
    """The scaled test input of one scale s: x itself for s == 1; otherwise x resized in float32 and padded with
    TTA_PAD.  Returned in float32."""
    if s == 1.0:
        return x
    (ch, cw), (ph, pw) = tta_sizes(x.shape[2], x.shape[3], s, gs)
    y = F.interpolate(x.float(), size=(ch, cw), mode="bilinear", align_corners=False)
    out = torch.full((x.shape[0], x.shape[1], ph, pw), TTA_PAD, dtype=torch.float32, device=x.device)
    out[..., :ch, :cw] = y
    return out


def yolox_forward_tta(sd, x, depth, num_classes, scales):
    """x [B,3,H,W] (BGR, 0..255) -> det_preds [B, A_tta, 5 + num_classes]: every scale's decoded output, boxes divided
    by the scale, concatenated in scale order."""
    outs = []
    for s in scales:
        d = yolox_forward(sd, tta_scale_input(x, s).to(x.dtype), depth, num_classes)
        outs.append(torch.cat([d[..., :4] / s, d[..., 4:]], -1))
    return torch.cat(outs, 1)
