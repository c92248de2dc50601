"""NumPy / cv2 / PIL restatement of read_data_train (core/gdrn_modeling/datasets/data_loader_online.py:311-581) for the
records of gdrnpp_bop2022_b200.train_batch: background replacement, the colour ops, the DZI crops.  Each op states the
reference call it restates and how it settles rounding; tests compare the CUDA pipeline with it bit for bit."""
import cv2
import numpy as np

from gdrnpp_bop2022_b200 import train_batch as TB

KIND = {v: k for k, v in TB.COLOR_OPS.items()}


# --------------------------------------------------------------------------------------------- colour ops
def coarse_dropout(img, cells):
    """imgaug CoarseDropout(p, size_percent): the per-image cell mask (cells, 1 = keep) upsampled with
    cv2.resize(INTER_NEAREST) to the image, multiplied into every channel.  Integer, no rounding."""
    H, W = img.shape[:2]
    m = cv2.resize(cells, (W, H), interpolation=cv2.INTER_NEAREST)
    return img * m[..., None]


def gaussian_blur(img, sigma):
    """imgaug blur_gaussian_ (cv2 backend): sigma <= 1e-3 leaves the image unchanged, else cv2.GaussianBlur with
    imgaug's ksize rule and BORDER_REFLECT_101; cv2's 8-bit fixed-point path settles the rounding."""
    if sigma <= TB.BLUR_EPS:
        return img
    k = TB.gaussian_ksize(sigma)
    return cv2.GaussianBlur(img, (k, k), sigmaX=sigma, sigmaY=sigma, borderType=cv2.BORDER_REFLECT_101)


def pil_luma(img):
    """PIL Image.convert("L") of the array seen as RGB: (R 19595 + G 38470 + B 7471 + 2^15) >> 16."""
    i = img.astype(np.int64)
    return ((i[..., 0] * 19595 + i[..., 1] * 38470 + i[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def pil_blend(deg, img, factor):
    """PIL ImagingBlend(degenerate, image, factor): deg + factor * (img - deg) in float32, truncated toward zero,
    clipped to [0, 255] (PIL.ImageEnhance._Enhance.enhance)."""
    a = np.float32(factor)
    t = deg.astype(np.float32) + a * (img.astype(np.int32) - deg.astype(np.int32)).astype(np.float32)
    return np.clip(np.trunc(t), 0, 255).astype(np.uint8)


def pil_smooth(img):
    """ImageFilter.SMOOTH ([1 1 1; 1 5 1; 1 1 1] / 13): float32 rows summed top to bottom, + 0.5, truncated; the
    one-pixel border is copied unfiltered."""
    out = img.copy()
    f = img.astype(np.float32)
    k1, k5 = np.float32(1) / np.float32(13), np.float32(5) / np.float32(13)
    H, W = img.shape[:2]
    ss = np.zeros((H - 2, W - 2, img.shape[2]), np.float32)
    for dy in (-1, 0, 1):
        kc = k5 if dy == 0 else k1
        r = f[1 + dy:H - 1 + dy]
        ss = ss + ((r[:, 0:W - 2] * k1 + r[:, 1:W - 1] * kc) + r[:, 2:W] * k1)
    out[1:-1, 1:-1] = np.clip(np.trunc(ss + np.float32(0.5)), 0, 255)
    return out


def enhance(img, kind, factor):
    """imgaug pillike.Enhance{Sharpness,Contrast,Brightness,Color} = PIL.ImageEnhance.<kind>(image).enhance(factor)."""
    if kind == "EnhanceSharpness":
        deg = pil_smooth(img)
    elif kind == "EnhanceContrast":
        deg = np.full_like(img, int(pil_luma(img).astype(np.float64).mean() + 0.5))
    elif kind == "EnhanceBrightness":
        deg = np.zeros_like(img)
    else:
        deg = np.repeat(pil_luma(img)[..., None], 3, axis=2)
    return pil_blend(deg, img, factor)


def _rint_clip(v):
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def add(img, values):
    """imgaug Add(value, per_channel): integer offset per channel, clipped."""
    return np.clip(img.astype(np.int32) + np.asarray(values[:3], np.int32), 0, 255).astype(np.uint8)


def invert(img, flags):
    """imgaug Invert(p, per_channel): 255 - v in the selected channels."""
    f = np.asarray(flags[:3], bool)
    return np.where(f, 255 - img, img).astype(np.uint8)


def multiply(img, factors):
    """imgaug Multiply(mul, per_channel): v * f in float64 (f the float32 draw), rounded half to even, clipped --
    cv2.multiply's saturate_cast."""
    return _rint_clip(img.astype(np.float64) * np.asarray(factors[:3], np.float32).astype(np.float64))


def philox4x32(ctr, k0, k1):
    """Philox4x32-10 of counters (ctr, 0, 0, 0) under key (k0, k1) -> four uint32 arrays."""
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
    x0 = ctr.astype(np.uint64)
    x1 = np.zeros_like(x0)
    x2 = np.zeros_like(x0)
    x3 = np.zeros_like(x0)
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = M0 * x0, M1 * x2
        y0 = (p1 >> np.uint64(32)) ^ x1 ^ np.uint64(k0)
        y2 = (p0 >> np.uint64(32)) ^ x3 ^ np.uint64(k1)
        x1, x3, x0, x2 = p1 & m32, p0 & m32, y0 & m32, y2 & m32
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return x0, x1, x2, x3


def gaussian_noise(img, scale, seed):
    """imgaug AdditiveGaussianNoise(scale, per_channel=True): v + N(0, scale) per pixel and channel, rounded half to
    even, clipped.  The normals: Box-Muller in float64 on Philox4x32-10 of (pixel index; seed), u = (r + 1) / 2^32."""
    H, W = img.shape[:2]
    k0, k1 = (int(s) & 0xFFFFFFFF for s in seed)
    r = philox4x32(np.arange(H * W, dtype=np.uint64), k0, k1)
    u = [(x.astype(np.float64) + 1.0) * 2.3283064365386963e-10 for x in r]
    ra, rb = np.sqrt(-2.0 * np.log(u[0])), np.sqrt(-2.0 * np.log(u[2]))
    ta, tb = 6.283185307179586 * u[1], 6.283185307179586 * u[3]
    z = np.stack([ra * np.cos(ta), ra * np.sin(ta), rb * np.cos(tb)], -1).reshape(H, W, 3)
    return _rint_clip(img.astype(np.float64) + np.float64(np.float32(scale)) * z)


def linear_contrast(img, alphas):
    """imgaug LinearContrast(alpha, per_channel): 127.5 + alpha (v - 127.5) in float64, rounded half to even, clipped."""
    a = np.asarray(alphas[:3], np.float32).astype(np.float64)
    return _rint_clip(127.5 + a * (img.astype(np.float64) - 127.5))


def grayscale(img, alpha):
    """imgaug Grayscale(alpha): cv2.cvtColor(COLOR_RGB2GRAY) of the array seen as RGB -- (R 9798 + G 19235 +
    B 3735 + 2^14) >> 15, the arithmetic of cv2's vectorised path, which covers whole rows of a 640-wide image (its
    scalar tail uses 14-bit weights) -- then gray * alpha + v * (1 - alpha) in float64, rounded half to even, clipped."""
    i = img.astype(np.int64)
    g = ((i[..., 0] * 9798 + i[..., 1] * 19235 + i[..., 2] * 3735 + (1 << 14)) >> 15).astype(np.float64)[..., None]
    a = np.float64(np.float32(alpha))
    return _rint_clip(g * a + img.astype(np.float64) * (1.0 - a))


def apply_op(img, kind, fpar, ipar, cells):
    """One colour op of the record (kind id, fpar, ipar, dropout cells) on a uint8 BGR image."""
    name = KIND.get(int(kind))
    if name is None:
        return img
    if name == "CoarseDropout":
        return coarse_dropout(img, cells)
    if name == "GaussianBlur":
        return gaussian_blur(img, float(fpar[0]))
    if name.startswith("Enhance"):
        return enhance(img, name, fpar[0])
    if name == "Add":
        return add(img, ipar)
    if name == "Invert":
        return invert(img, ipar)
    if name == "Multiply":
        return multiply(img, fpar)
    if name == "AdditiveGaussianNoise":
        return gaussian_noise(img, fpar[0], ipar[:2].view(np.uint32))
    if name == "LinearContrast":
        return linear_contrast(img, fpar)
    return grayscale(img, fpar[0])


# --------------------------------------------------------------------------------------------- background
def trunc_window(mask, side, u):
    """trunc_mask (base_data_loader.py:454-478) with random.random() = side's draw and random.uniform(a, b) =
    a + (b - a) * u, int() truncation -> keep window (row0, row1, col0, col1)."""
    H, W = mask.shape
    k = [0, H, 0, W]
    if side in (0, 1, 2, 3):
        nz = np.nonzero(mask)
        x1, y1 = np.min(nz, axis=1)
        x2, y2 = np.max(nz, axis=1)
        lo, hi = (float(x1), float(x2)) if side < 2 else (float(y1), float(y2))
        c = 0.5 * (lo + hi)
        a, e = (c, hi) if side & 1 else (lo, c)
        k[side] = int(a + (e - a) * u)
    return k


def background(bg, H, W):
    """get_bg_image (base_data_loader.py:480-551): the top-left crop, resize_short_edge (cv2.resize with fx = fy),
    placed top-left on a zero canvas."""
    ch, cw, rh, rw, _ = TB.bg_layout(bg.shape[:2], H, W)
    crop = bg[:ch, :cw]
    s_min, s_max = min(ch, cw), max(ch, cw)
    scale = float(min(H, W)) / float(s_min)
    if np.round(scale * s_max) > max(H, W):
        scale = float(max(H, W)) / float(s_max)
    r = cv2.resize(crop, None, None, fx=scale, fy=scale, interpolation=cv2.INTER_LINEAR)
    out = np.zeros((H, W, 3), np.uint8)
    out[:r.shape[0], :r.shape[1]] = r
    return out


# --------------------------------------------------------------------------------------------- crops
def affine(center, scale, res):
    """get_affine_transform(center, (scale, scale), 0, (res, res)) as cv2.getAffineTransform of its float32 points."""
    c = np.asarray(center, np.float64)
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0] = c
    src[1] = c + np.array([0, scale * -0.5])
    d = src[0] - src[1]
    src[2] = src[1] + np.array([-d[1], d[0]], np.float32)
    dst[0] = [res * 0.5, res * 0.5]
    dst[1] = dst[0] + np.array([0, res * -0.5], np.float32)
    d = dst[0] - dst[1]
    dst[2] = dst[1] + np.array([-d[1], d[0]], np.float32)
    return cv2.getAffineTransform(src, dst)


def coord_2d(H, W):
    """get_2d_coord_np(W, H).transpose(1, 2, 0): x, y in [0, 1) float32."""
    x = np.linspace(0, 1, W, endpoint=False, dtype=np.float32)
    y = np.linspace(0, 1, H, endpoint=False, dtype=np.float32)
    xy = np.stack(np.meshgrid(x, y), -1)
    return np.ascontiguousarray(xy.astype(np.float32))


def roi_geometry(cfg, ts, rec):
    """The box arithmetic of read_data_train, restated from the reference for the records: -> center [n,2],
    scale [n], wh [n,2], trans_ratio [n,3] in float64.
      registrar (datasets/ycbv_pbr.py:124-151): K float32, t = cam_t_m2c float32 / 1000, centroid_2d =
        ((K @ t.T).T)[:2] / ((K @ t.T).T)[2];
      transform_instance_annotations: BoxMode XYWH -> XYXY (x2 = x + w), the identity resize, "bbox" clipped to
        [0, W] x [0, H];
      data_loader_online.py:466-482: VISIB takes "bbox", AMODAL_CLIP clips "bbox_obj" to the image;
      base_data_loader.py:188-231 aug_bbox_DZI with the record's scale / shift ratios, then min(scale, max(H, W));
      data_loader_online.py:481-580: bw, bh = max(x2 - x1, 1), max(y2 - y1, 1), resize_ratio = out_res / scale,
        trans_ratio = ((c - center) / (bw, bh), t_z / resize_ratio)."""
    im_H, im_W = ts.im_size
    out_res = TB.cfg_get(cfg, "MODEL.POSE_NET.OUTPUT_RES", 64)
    bbox_type = str(TB.cfg_get(cfg, "MODEL.BBOX_TYPE", "VISIB")).lower()
    dzi_type = str(TB.cfg_get(cfg, "INPUT.DZI_TYPE", "uniform")).lower()
    dzi_pad_scale = TB.cfg_get(cfg, "INPUT.DZI_PAD_SCALE", 1.0)
    n = len(rec["index"])
    out = {"center": np.zeros((n, 2)), "scale": np.zeros(n), "wh": np.zeros((n, 2)), "trans_ratio": np.zeros((n, 3))}
    for b in range(n):
        s = ts.samples[rec["index"][b]]
        K, t = np.asarray(s["K"], np.float32), np.asarray(s["t"], np.float32)
        proj = (K @ t.T).T
        obj_center = proj[:2] / proj[2]
        x, y, w, h = s["bbox_visib"]
        bbox = np.array([x, y, x + w, y + h], np.float64).clip(min=0)
        bbox = np.minimum(bbox, [im_W, im_H, im_W, im_H])
        if bbox_type == "visib":
            bbox_xyxy = bbox
        else:
            x, y, w, h = s["bbox_obj"]
            ax1, ay1, ax2, ay2 = np.array([x, y, x + w, y + h], np.float64)
            bbox_xyxy = np.array([max(ax1, 0), max(ay1, 0), min(ax2, im_W), min(ay2, im_H)])
        x1, y1, x2, y2 = bbox_xyxy.copy()
        cx, cy = 0.5 * (x1 + x2), 0.5 * (y1 + y2)
        bh, bw = y2 - y1, x2 - x1
        if dzi_type == "uniform":
            scale_ratio, shift_ratio = rec["dzi_scale"][b], rec["dzi_shift"][b]
            bbox_center = np.array([cx + bw * shift_ratio[0], cy + bh * shift_ratio[1]])
            scale = max(y2 - y1, x2 - x1) * scale_ratio * dzi_pad_scale
        else:
            bbox_center = np.array([cx, cy])
            scale = max(y2 - y1, x2 - x1)
        scale = min(scale, max(im_H, im_W)) * 1.0
        bw, bh = max(bbox_xyxy[2] - bbox_xyxy[0], 1), max(bbox_xyxy[3] - bbox_xyxy[1], 1)
        resize_ratio = out_res / scale
        z_ratio = t[2] / resize_ratio
        delta_c = obj_center - bbox_center
        out["center"][b], out["scale"][b], out["wh"][b] = bbox_center, scale, (bw, bh)
        out["trans_ratio"][b] = (delta_c[0] / bw, delta_c[1] / bh, z_ratio)
    return out


def replay(cfg, ts, bg_paths, rec):
    """The per-sample images of the records: -> dict with image [n,H,W,3] (after background and colour),
    roi_img, roi_coord_2d, roi_mask_trunc / visib / full (before mask_obj) and counts [n,2]."""
    H, W = ts.im_size
    in_res = int(TB.cfg_get(cfg, "MODEL.POSE_NET.INPUT_RES", 256))
    out_res = int(TB.cfg_get(cfg, "MODEL.POSE_NET.OUTPUT_RES", 64))
    mean = np.asarray(TB.cfg_get(cfg, "MODEL.PIXEL_MEAN", [0.0, 0.0, 0.0]), np.float64).reshape(3, 1, 1)
    std = np.asarray(TB.cfg_get(cfg, "MODEL.PIXEL_STD", [255.0, 255.0, 255.0]), np.float64).reshape(3, 1, 1)
    imgs, mvs, mfs, bgs = TB.decode(ts, bg_paths, rec)
    geo = roi_geometry(cfg, ts, rec)
    c2d = coord_2d(H, W)
    n = len(rec["index"])
    out = {k: [] for k in ("image", "roi_img", "roi_coord_2d", "roi_mask_trunc", "roi_mask_visib", "roi_mask_full",
                           "counts")}
    for b in range(n):
        im, mv, mf = imgs[b].copy(), mvs[b], mfs[b]
        keep = [0, H, 0, W]
        if rec["do_bg"][b]:
            keep = trunc_window(mv, int(rec["trunc_side"][b]), float(rec["trunc_u"][b]))
            m = np.zeros_like(mv, bool)
            m[keep[0]:keep[1], keep[2]:keep[3]] = mv[keep[0]:keep[1], keep[2]:keep[3]] > 0
            bg = background(bgs[b], H, W)
            im[~m] = bg[~m]
        if rec["do_color"][b]:
            for s in range(rec["kind_at"].shape[1]):
                im = apply_op(im, rec["kind_at"][b, s], rec["fpar"][b, s], rec["ipar"][b, s], rec["cells"][b])
        trunc = np.zeros_like(mv, np.float32)
        trunc[keep[0]:keep[1], keep[2]:keep[3]] = 1
        trunc = mv.astype(np.float32) * trunc
        Mi, Mo = affine(geo["center"][b], geo["scale"][b], in_res), affine(geo["center"][b], geo["scale"][b], out_res)
        roi = cv2.warpAffine(im, Mi, (in_res, in_res), flags=cv2.INTER_LINEAR).transpose(2, 0, 1)
        out["roi_img"].append(((roi - mean) / std).astype(np.float32))
        out["roi_coord_2d"].append(cv2.warpAffine(c2d, Mo, (out_res, out_res), flags=cv2.INTER_LINEAR).transpose(2, 0, 1))
        crops = [cv2.warpAffine(m.astype(np.float32), Mo, (out_res, out_res), flags=cv2.INTER_NEAREST)
                 for m in (trunc, mv, mf)]
        for key, c in zip(("roi_mask_trunc", "roi_mask_visib", "roi_mask_full"), crops):
            out[key].append(c)
        out["counts"].append([int(crops[0].sum()), int(crops[1].sum())])
        out["image"].append(im)
    return {k: np.stack(v) for k, v in out.items()}
