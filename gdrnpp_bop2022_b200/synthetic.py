"""Seeded synthetic weights and ROI batches (SURVEY.md §8d, configs 1-5).

There is no network for datasets or checkpoints, so both sides of every parity
test (CUDA path and oracle) consume the ``state_dict`` and the batch made here.

Weight distribution: the reference's own random init is numerically degenerate
(ConvNeXt layer-scale gamma = 1e-6, head convs N(0, 1e-3); SURVEY.md §7 "hard
parts"), which would make R|t parity pure noise.  We use a variance-preserving
init instead (He-scaled convs/linears, gamma ~ U(0.1, 0.4), norm affine params
perturbed around identity) and record it here; key names and shapes are exactly
those of a reference checkpoint (SURVEY.md Appendix A).
"""
import math

import numpy as np
import torch

CONVNEXT_ARCH = {
    "convnext_tiny": ((3, 3, 9, 3), (96, 192, 384, 768)),
    "convnext_small": ((3, 3, 27, 3), (96, 192, 384, 768)),
    "convnext_base": ((3, 3, 27, 3), (128, 256, 512, 1024)),
}

YCBV_K = ((1066.778, 0.0, 312.9869), (0.0, 1067.487, 241.3109), (0.0, 0.0, 1.0))  # ref/ycbv.py:89


def state_dict_shapes(arch="convnext_base", num_classes=21, num_regions=64):
    """{key: shape} of a reference checkpoint (SURVEY.md Appendix A) without materialising any weights."""
    depths, dims = CONVNEXT_ARCH[arch]
    sh = {}

    def norm(prefix, c):
        sh[prefix + ".weight"] = (c,)
        sh[prefix + ".bias"] = (c,)

    b = "backbone."
    sh[b + "stem_0.weight"] = (dims[0], 3, 4, 4)
    sh[b + "stem_0.bias"] = (dims[0],)
    norm(b + "stem_1", dims[0])
    for s in range(4):
        C = dims[s]
        if s > 0:
            norm(b + f"stages_{s}.downsample.0", dims[s - 1])
            sh[b + f"stages_{s}.downsample.1.weight"] = (C, dims[s - 1], 2, 2)
            sh[b + f"stages_{s}.downsample.1.bias"] = (C,)
        for i in range(depths[s]):
            p = b + f"stages_{s}.blocks.{i}."
            sh[p + "conv_dw.weight"] = (C, 1, 7, 7)
            sh[p + "conv_dw.bias"] = (C,)
            norm(p + "norm", C)
            sh[p + "mlp.fc1.weight"] = (4 * C, C)
            sh[p + "mlp.fc1.bias"] = (4 * C,)
            sh[p + "mlp.fc2.weight"] = (C, 4 * C)
            sh[p + "mlp.fc2.bias"] = (C,)
            sh[p + "gamma"] = (C,)
    h = "geo_head_net."
    sh[h + "features.0.weight"] = (dims[3], 256, 3, 3)
    norm(h + "features.1", 256)
    for i in (3, 4, 6, 7, 9, 10):
        sh[h + f"features.{i}.conv.weight"] = (256, 256, 3, 3)
        norm(h + f"features.{i}.gn", 256)
    out_dim = num_classes * (2 + 3 + num_regions + 1)
    sh[h + "out_layer.weight"] = (out_dim, 256, 1, 1)
    sh[h + "out_layer.bias"] = (out_dim,)
    p = "pnp_net."
    n_in = 3 + 2 + num_regions
    for j, i in enumerate((0, 3, 6)):
        sh[p + f"features.{i}.weight"] = (128, n_in if j == 0 else 128, 3, 3)
        norm(p + f"features.{i+1}", 128)
    sh[p + "fc1.weight"] = (1024, 8192)
    sh[p + "fc1.bias"] = (1024,)
    sh[p + "fc2.weight"] = (256, 1024)
    sh[p + "fc2.bias"] = (256,)
    sh[p + "fc_r.weight"] = (6, 256)
    sh[p + "fc_r.bias"] = (6,)
    sh[p + "fc_t.weight"] = (3, 256)
    sh[p + "fc_t.bias"] = (3,)
    return sh


def make_state_dict(arch="convnext_base", num_classes=21, num_regions=64, seed=0):
    """fp32 state_dict with reference key names: backbone.* / geo_head_net.* / pnp_net.*"""
    g = torch.Generator().manual_seed(seed)
    depths, dims = CONVNEXT_ARCH[arch]
    sd = {}

    def randn(shape, std):
        return torch.randn(shape, generator=g) * std

    def uni(shape, lo, hi):
        return torch.rand(shape, generator=g) * (hi - lo) + lo

    def norm_affine(prefix, c):
        sd[prefix + ".weight"] = uni((c,), 0.8, 1.2)
        sd[prefix + ".bias"] = randn((c,), 0.05)

    b = "backbone."
    sd[b + "stem_0.weight"] = randn((dims[0], 3, 4, 4), 1.0 / math.sqrt(48) * 2.0)
    sd[b + "stem_0.bias"] = randn((dims[0],), 0.1)
    norm_affine(b + "stem_1", dims[0])
    for s in range(4):
        C = dims[s]
        if s > 0:
            norm_affine(b + f"stages_{s}.downsample.0", dims[s - 1])
            sd[b + f"stages_{s}.downsample.1.weight"] = randn((C, dims[s - 1], 2, 2), 1.0 / math.sqrt(4 * dims[s - 1]))
            sd[b + f"stages_{s}.downsample.1.bias"] = randn((C,), 0.05)
        for i in range(depths[s]):
            p = b + f"stages_{s}.blocks.{i}."
            sd[p + "conv_dw.weight"] = randn((C, 1, 7, 7), 1.0 / 7.0)
            sd[p + "conv_dw.bias"] = randn((C,), 0.05)
            norm_affine(p + "norm", C)
            sd[p + "mlp.fc1.weight"] = randn((4 * C, C), 1.0 / math.sqrt(C))
            sd[p + "mlp.fc1.bias"] = randn((4 * C,), 0.05)
            sd[p + "mlp.fc2.weight"] = randn((C, 4 * C), math.sqrt(2.0) / math.sqrt(4 * C))
            sd[p + "mlp.fc2.bias"] = randn((C,), 0.05)
            sd[p + "gamma"] = uni((C,), 0.1, 0.4)

    h = "geo_head_net."
    in_dim = dims[3]
    sd[h + "features.0.weight"] = randn((in_dim, 256, 3, 3), math.sqrt(2.0) / math.sqrt(in_dim * 9 / 4))
    norm_affine(h + "features.1", 256)
    for i in (3, 4, 6, 7, 9, 10):
        sd[h + f"features.{i}.conv.weight"] = randn((256, 256, 3, 3), math.sqrt(2.0) / math.sqrt(256 * 9))
        norm_affine(h + f"features.{i}.gn", 256)
    out_dim = num_classes * (2 + 3 + num_regions + 1)
    sd[h + "out_layer.weight"] = randn((out_dim, 256, 1, 1), 1.0 / math.sqrt(256))
    sd[h + "out_layer.bias"] = randn((out_dim,), 0.1)
    # xyz outputs are expected in [0,1] by the PnP denormalisation: centre them at 0.5
    sd[h + "out_layer.bias"][2 * num_classes : 5 * num_classes] += 0.5
    sd[h + "out_layer.weight"][2 * num_classes : 5 * num_classes] *= 0.25

    p = "pnp_net."
    n_in = 3 + 2 + num_regions
    for j, i in enumerate((0, 3, 6)):
        cin = n_in if j == 0 else 128
        sd[p + f"features.{i}.weight"] = randn((128, cin, 3, 3), math.sqrt(2.0) / math.sqrt(cin * 9))
        norm_affine(p + f"features.{i+1}", 128)
    sd[p + "fc1.weight"] = randn((1024, 8192), math.sqrt(2.0) / math.sqrt(8192))
    sd[p + "fc1.bias"] = randn((1024,), 0.05)
    sd[p + "fc2.weight"] = randn((256, 1024), math.sqrt(2.0) / math.sqrt(1024))
    sd[p + "fc2.bias"] = randn((256,), 0.05)
    sd[p + "fc_r.weight"] = randn((6, 256), 1.0 / math.sqrt(256))
    sd[p + "fc_r.bias"] = randn((6,), 0.3)
    sd[p + "fc_t.weight"] = randn((3, 256), 0.2 / math.sqrt(256))
    sd[p + "fc_t.bias"] = torch.tensor([0.0, 0.0, 1.0]) + randn((3,), 0.02)
    return sd


def make_batch(B=64, seed=0, num_classes=21, im_w=640, im_h=480, in_res=256, out_res=64):
    """Synthetic ROI batch with the tensor contract of datasets/data_loader.py:647-818
    (roi_img in [0,1) because PIXEL_MEAN 0 / PIXEL_STD 255)."""
    g = torch.Generator().manual_seed(1000 + seed)
    roi_img = torch.rand((B, 3, in_res, in_res), generator=g)
    roi_classes = torch.randint(0, num_classes, (B,), generator=g)
    cx = torch.rand((B,), generator=g) * im_w
    cy = torch.rand((B,), generator=g) * im_h
    bw = torch.rand((B,), generator=g) * 160 + 40
    bh = torch.rand((B,), generator=g) * 160 + 40
    scale = torch.clamp(torch.maximum(bw, bh) * 1.5, max=float(max(im_w, im_h)))
    resize_ratios = out_res / scale
    u = torch.arange(out_res, dtype=torch.float32)
    # affine crop: dst pixel u <-> src = c + (u - out_res/2) * scale/out_res (data_utils.py:136-184)
    sx = cx[:, None] + (u[None, :] - out_res / 2) * (scale[:, None] / out_res)
    sy = cy[:, None] + (u[None, :] - out_res / 2) * (scale[:, None] / out_res)
    gx = torch.where((sx >= 0) & (sx <= im_w - 1), sx / im_w, torch.zeros_like(sx))
    gy = torch.where((sy >= 0) & (sy <= im_h - 1), sy / im_h, torch.zeros_like(sy))
    coord = torch.stack(
        [gx[:, None, :].expand(B, out_res, out_res), gy[:, :, None].expand(B, out_res, out_res)], dim=1
    ).contiguous()
    roi_cams = torch.tensor(YCBV_K, dtype=torch.float32)[None].repeat(B, 1, 1)
    extents = torch.rand((B, 3), generator=g) * 0.2 + 0.05
    return {
        "roi_img": roi_img,
        "roi_classes": roi_classes,
        "roi_coord_2d": coord,
        "roi_cams": roi_cams,
        "roi_centers": torch.stack([cx, cy], dim=1),
        "roi_whs": torch.stack([bw, bh], dim=1),
        "resize_ratios": resize_ratios,
        "roi_extents": extents,
    }


def make_icosphere_mesh(subdiv=3, extent=(0.1, 0.1, 0.1)):
    """Unit icosphere scaled to ``extent`` (full widths, metres): verts [V,3] f32, faces [F,3] i32."""
    t = (1.0 + math.sqrt(5.0)) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
         (8, 6, 7), (9, 8, 1)]
    v = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdiv):
        cache = {}
        nf = []

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = v[a] + v[b]
                v.append(m / np.linalg.norm(m))
                cache[key] = len(v) - 1
            return cache[key]

        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    verts = np.array(v, dtype=np.float64) * (np.array(extent, dtype=np.float64) / 2.0)
    return verts.astype(np.float32), np.array(f, dtype=np.int32)


def make_yolox_state_dict(forward, depth=0.33, width=0.25, num_classes=8, seed=0, calib_hw=(640, 640), calib_batch=2,
                          device="cpu", target_conf=0.5, keep_frac=0.03, bn_gain=(0.4, 0.6), var_floor=1.0, bn_bias_std=1.0):
    """Seeded YOLOX weights with the reference's state-dict keys (unfused, BatchNorm buffers included).

    Random weights through a hundred folded conv layers would explode or vanish, so every BatchNorm's running mean and
    variance are set from the statistics of its own input on a seeded calibration batch (``calib_batch`` images of ``calib_hw``; calibrate at the input size that will be
    run: the SPP pools and the zero-padded borders make the statistics depend on the map size),
    passed through ``forward`` (a float64 functional restatement of the network, ``forward(sd, x, depth,
    num_classes, on_conv=...)`` calling ``on_conv(prefix, conv_out)`` before each BatchNorm, as the test oracle does)
    layer by layer: activations stay O(1) as in a trained
    network.  Each variance is floored at its layer's mean variance, so that channels that are nearly constant over the
    calibration images do not amplify other inputs.  Conv weights N(0, 1/fan_in) (box predictions x 0.25), BatchNorm
    weight U(0.4, 0.6) and bias N(0, 1): with the biases large against the weights the random network sits in the
    ordered regime, where a rounding error shrinks from layer to layer instead of growing (with weight U(0.8, 1.2) and
    bias N(0, 0.2) the fp32 forward of YOLOX-X already misses the fp64 one by pixels).  The prediction biases
    start from the head's prior_prob = 0.01 init and are then shifted so that on the calibration batch the median class
    logit reaches sigmoid 0.9 and about ``keep_frac`` of the anchors score at least ``target_conf``: a few hundred of
    the 8400 anchors of a 640 x 640 image clear such a threshold."""
    from .yolox_model import YOLOX

    shapes = {k: tuple(v.shape) for k, v in YOLOX(depth, width, num_classes, max_batch=1).state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, s in shapes.items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros((), dtype=torch.int64)
        elif len(s) == 4:
            sd[k] = torch.randn(s, generator=g, dtype=torch.float64) * math.sqrt(1.0 / (s[1] * s[2] * s[3]))
            if ".reg_preds." in k:
                sd[k] *= 0.25
        elif k.endswith("bn.weight"):
            sd[k] = torch.rand(s, generator=g, dtype=torch.float64) * (bn_gain[1] - bn_gain[0]) + bn_gain[0]
        elif k.endswith("running_var"):
            sd[k] = torch.ones(s, dtype=torch.float64)
        elif k.endswith("running_mean"):
            sd[k] = torch.zeros(s, dtype=torch.float64)
        elif ".obj_preds." in k or ".cls_preds." in k:
            sd[k] = torch.full(s, -math.log((1 - 0.01) / 0.01), dtype=torch.float64)
        elif ".reg_preds." in k:
            sd[k] = torch.zeros(s, dtype=torch.float64)
        else:
            sd[k] = torch.randn(s, generator=g, dtype=torch.float64) * bn_bias_std
    dev = torch.device(device)
    sd = {k: v.to(dev) for k, v in sd.items()}
    x = torch.rand((calib_batch, 3) + tuple(calib_hw), generator=g, dtype=torch.float64).to(dev) * 255

    def calibrate(prefix, y):
        sd[prefix + ".bn.running_mean"] = y.mean((0, 2, 3))
        v = y.var((0, 2, 3), unbiased=False)
        # floor: a channel that is nearly constant over noise images must not amplify another image's offsets
        sd[prefix + ".bn.running_var"] = v + var_floor * v.mean()

    with torch.no_grad():
        forward(sd, x, depth, num_classes, on_conv=calibrate)
        for k in range(3):   # logits without the prior
            sd[f"head.obj_preds.{k}.bias"].zero_()
            sd[f"head.cls_preds.{k}.bias"].zero_()
        d = forward(sd, x, depth, num_classes)
        logit = lambda p: torch.log(p) - torch.log1p(-p)  # noqa: E731
        zc = logit(d[..., 5:].clamp(1e-12, 1 - 1e-12)).flatten()
        zo = logit(d[..., 4].clamp(1e-12, 1 - 1e-12)).flatten()
        b_c = math.log(9.0) - torch.quantile(zc, 0.5).item()
        q = min(target_conf / 0.9, 0.999)
        b_o = math.log(q / (1 - q)) - torch.quantile(zo, 1 - keep_frac).item()
        for k in range(3):
            sd[f"head.obj_preds.{k}.bias"].fill_(b_o)
            sd[f"head.cls_preds.{k}.bias"].fill_(b_c)
    return {k: (v.float() if v.is_floating_point() else v).cpu() for k, v in sd.items()}


def write_bop_tree(root, dataset="ycbv", num_images=12, num_scenes=2, H=480, W=640, dets_per_image=6, seed=0, gray=False,
                   obj_ids=None, with_depth=True):
    """A small BOP test split under ``root`` (the reference's ``datasets/`` directory): BOP_DATASETS/<dataset>/ with
    test_targets_bop19.json, test/<scene>/{rgb|gray, depth, scene_camera.json, scene_gt.json, scene_gt_info.json},
    models_eval/ (box meshes in mm + models_info.json) and test/test_bboxes/dets.json (detections, XYWH boxes around the
    ground-truth objects, some partly outside the image).  Colour images are random BGR PNGs (``gray``: 8-bit TIFs in
    gray/, as ITODD), depth 16-bit PNGs of a tilted plane.  -> path of the detection file relative to ``root``, as "datasets/..."."""
    import json
    import os

    import cv2

    from .ply import save_ply

    rng = np.random.RandomState(seed)
    base = os.path.join(root, "BOP_DATASETS", dataset)
    split = os.path.join(base, "test_primesense" if dataset in ("tless", "hb") else "test")
    models = os.path.join(base, "models_eval")
    os.makedirs(models, exist_ok=True)
    obj_ids = list(obj_ids or range(1, 22))
    info = {}
    faces = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                      [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    for o in obj_ids:
        half = rng.uniform(20, 60, 3)
        pts = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float32) * half
        save_ply(os.path.join(models, "obj_{:06d}.ply".format(o)), pts, faces)
        info[str(o)] = {"diameter": float(2 * np.linalg.norm(half)), "min_x": float(-half[0]), "min_y": float(-half[1]),
                        "min_z": float(-half[2]), "size_x": float(2 * half[0]), "size_y": float(2 * half[1]),
                        "size_z": float(2 * half[2])}
    with open(os.path.join(models, "models_info.json"), "w") as f:
        json.dump(info, f)
    targets, dets = [], {}
    color_dir, ext = ("gray", ".tif") if gray else ("rgb", ".png")
    per_scene = -(-num_images // num_scenes)
    for s in range(num_scenes):
        scene_id = s + 1
        sdir = os.path.join(split, "{:06d}".format(scene_id))
        os.makedirs(os.path.join(sdir, color_dir), exist_ok=True)
        os.makedirs(os.path.join(sdir, "depth"), exist_ok=True)
        cams, gts, gt_infos = {}, {}, {}
        for k in range(min(per_scene, num_images - s * per_scene)):
            im_id = 3 * k + 1
            f = W * rng.uniform(0.9, 1.1)
            K = [f, 0.0, W / 2 + rng.uniform(-5, 5), 0.0, f, H / 2 + rng.uniform(-5, 5), 0.0, 0.0, 1.0]
            depth_scale = float(rng.choice([0.1, 1.0]))
            cams[str(im_id)] = {"cam_K": K, "depth_scale": depth_scale}
            im = rng.randint(0, 256, (H, W) if gray else (H, W, 3)).astype(np.uint8)
            cv2.imwrite(os.path.join(sdir, color_dir, "{:06d}{}".format(im_id, ext)), im)
            yy, xx = np.mgrid[0:H, 0:W]   # a tilted plane 0.8-1.2 m away with a few mm of noise, in depth_scale units
            depth_mm = 800 + 300 * xx / W + 100 * yy / H + rng.uniform(0, 5, (H, W))
            cv2.imwrite(os.path.join(sdir, "depth", "{:06d}{}".format(im_id, ext)),
                        np.round(depth_mm / depth_scale).astype(np.uint16))
            gts[str(im_id)], gt_infos[str(im_id)], cur = [], [], []
            for j, o in enumerate(rng.choice(obj_ids, min(dets_per_image, len(obj_ids)), replace=False)):
                o = int(o)
                R = cv2.Rodrigues(rng.uniform(-1, 1, 3))[0]
                t = np.array([rng.uniform(-150, 150), rng.uniform(-100, 100), rng.uniform(600, 1200)])
                gts[str(im_id)].append({"obj_id": o, "cam_R_m2c": R.reshape(-1).tolist(), "cam_t_m2c": t.tolist()})
                u, v = f * t[0] / t[2] + K[2], f * t[1] / t[2] + K[5]
                bw, bh = rng.uniform(0.3, 200), rng.uniform(0.3, 200)
                x, y = u - bw / 2 + rng.uniform(-100, 100) * (j == 0), v - bh / 2
                gt_infos[str(im_id)].append({"bbox_obj": [int(x), int(y), int(bw), int(bh)],
                                             "bbox_visib": [int(x), int(y), int(bw), int(bh)], "px_count_all": 1000,
                                             "px_count_valid": 1000, "px_count_visib": 900, "visib_fract": 0.9})
                cur.append({"obj_id": o, "bbox_est": [float(x), float(y), float(bw), float(bh)],
                            "score": float(np.round(rng.uniform(0.05, 1.0), 2)), "time": 0.01})
            dets["{}/{}".format(scene_id, im_id)] = cur
            for o in sorted({g["obj_id"] for g in gts[str(im_id)]}):
                targets.append({"scene_id": scene_id, "im_id": im_id, "obj_id": o,
                                "inst_count": sum(g["obj_id"] == o for g in gts[str(im_id)])})
        for name, content in (("scene_camera.json", cams), ("scene_gt.json", gts), ("scene_gt_info.json", gt_infos)):
            with open(os.path.join(sdir, name), "w") as f:
                json.dump(content, f)
    with open(os.path.join(base, "test_targets_bop19.json"), "w") as f:
        json.dump(targets, f)
    os.makedirs(os.path.join(split, "test_bboxes"), exist_ok=True)
    with open(os.path.join(split, "test_bboxes", "dets.json"), "w") as f:
        json.dump(dets, f)
    return "datasets/" + os.path.relpath(os.path.join(split, "test_bboxes", "dets.json"), root)
