"""GDRN training batches built on the GPU: the reference's GDRN_Online_DatasetFromList.read_data_train
(core/gdrn_modeling/datasets/data_loader_online.py:311-581) for every sample of a batch, then batch_data_train_online
(core/gdrn_modeling/engine/engine_utils.py:76-210).

Every random choice is drawn on the host, from one numpy Generator per batch, into a fixed-layout record per sample
(``Sampler.draw``).  The device work (csrc/train_aug.cu) is a deterministic function of (images, records): background
composite with the truncated foreground, the colour-augmentation program one batched pass per position of its random
order, the DZI-jittered ROI crops; then online_targets.render_roi_targets renders xyz / region / mask_obj.  The only
synchronisation in a batch is one device-to-host copy of the ROIs' trunc / visib pixel counts, which drives the
reference's redraw of samples whose cropped masks have fewer than 32 pixels.

    python -m gdrnpp_bop2022_b200.train_batch compute_fps --dataset D [--datasets-root R]
writes <models>/fps_points.pkl, the farthest-point-sampling points the region targets need.
"""
import argparse
import ast
import json
import math
import os
import pickle
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib
from .gdrn_evaluator import _resize_shortest_edge_size, cfg_get, read_image, resolve_path
from .gt_info import models_path, plan_split, split_params

GdrnError = _lib.GdrnError

# --------------------------------------------------------------------------------------------- colour augmentation
# kind ids shared with csrc/train_aug.cu
COLOR_OPS = {"CoarseDropout": 0, "GaussianBlur": 1, "EnhanceSharpness": 2, "EnhanceContrast": 3, "EnhanceBrightness": 4,
             "EnhanceColor": 5, "Add": 6, "Invert": 7, "Multiply": 8, "AdditiveGaussianNoise": 9, "LinearContrast": 10,
             "Grayscale": 11}
N_FPAR, N_IPAR = 4, 12
MAX_BLUR_TAPS = N_IPAR - 1   # GaussianBlur's ipar: ksize, then the taps
BLUR_EPS = 1e-3   # imgaug's blur_gaussian_: sigma <= eps leaves the image unchanged
# each op's keyword names in positional order, and the defaults imgaug gives them
_OP_ARGS = {
    "CoarseDropout": (("p", 0.02), ("size_px", None), ("size_percent", None), ("per_channel", False), ("min_size", 3)),
    "GaussianBlur": (("sigma", (0.0, 3.0)),),
    "EnhanceSharpness": (("factor", (0.0, 2.0)),),
    "EnhanceContrast": (("factor", (0.5, 1.5)),),
    "EnhanceBrightness": (("factor", (0.5, 1.5)),),
    "EnhanceColor": (("factor", (0.0, 3.0)),),
    "Add": (("value", (-20, 20)), ("per_channel", False)),
    "Invert": (("p", 1), ("per_channel", False), ("min_value", None), ("max_value", None)),
    "Multiply": (("mul", (0.8, 1.2)), ("per_channel", False)),
    "AdditiveGaussianNoise": (("loc", 0), ("scale", (0, 15)), ("per_channel", False)),
    "LinearContrast": (("alpha", (0.6, 1.4)), ("per_channel", False)),
    "Grayscale": (("alpha", 1),),
}


def _literal(node, code):
    try:
        return ast.literal_eval(node)
    except ValueError:
        raise GdrnError(f"COLOR_AUG_CODE: argument {ast.unparse(node)!r} is not a literal ({code!r})") from None


def _call_name(node):
    f = node.func
    return f.attr if isinstance(f, ast.Attribute) else (f.id if isinstance(f, ast.Name) else None)


def _parse_op(node, code):
    if not isinstance(node, ast.Call):
        raise GdrnError(f"COLOR_AUG_CODE: expected an augmenter call, got {ast.unparse(node)!r}")
    name = _call_name(node)
    prob = 1.0
    if name == "Sometimes":
        if len(node.args) != 2 or node.keywords:
            raise GdrnError(f"COLOR_AUG_CODE: Sometimes takes (p, augmenter): {ast.unparse(node)!r}")
        prob = float(_literal(node.args[0], code))
        node = node.args[1]
        if not isinstance(node, ast.Call):
            raise GdrnError(f"COLOR_AUG_CODE: expected an augmenter call, got {ast.unparse(node)!r}")
        name = _call_name(node)
    if name not in _OP_ARGS:
        raise GdrnError(f"COLOR_AUG_CODE: augmenter {name!r} is not supported (supported: {', '.join(_OP_ARGS)})")
    spec = _OP_ARGS[name]
    kw = {k: d for k, d in spec}
    if len(node.args) > len(spec):
        raise GdrnError(f"COLOR_AUG_CODE: too many arguments for {name}")
    for (k, _), a in zip(spec, node.args):
        kw[k] = _literal(a, code)
    for k in node.keywords:
        if k.arg not in kw:
            raise GdrnError(f"COLOR_AUG_CODE: {name} argument {k.arg!r} is not supported")
        kw[k.arg] = _literal(k.value, code)
    for k, v in kw.items():
        if isinstance(v, list):
            raise GdrnError(f"COLOR_AUG_CODE: {name}({k}={v!r}): lists (a choice of values) are not supported")
        if isinstance(v, tuple) and (len(v) != 2 or not all(isinstance(x, (int, float)) for x in v)):
            raise GdrnError(f"COLOR_AUG_CODE: {name}({k}={v!r}): a range must be a pair of numbers (low, high)")
    if name == "CoarseDropout" and (kw["size_percent"] is None or kw["size_px"] is not None or kw["per_channel"]):
        raise GdrnError("COLOR_AUG_CODE: CoarseDropout is supported with size_percent and per_channel=False only")
    if name == "CoarseDropout" and not isinstance(kw["size_percent"], (int, float)):
        raise GdrnError(f"COLOR_AUG_CODE: CoarseDropout(size_percent={kw['size_percent']!r}): only a fixed size_percent "
                        "is supported (the cell grid is one size per batch)")
    if name == "GaussianBlur":
        s = kw["sigma"]
        lo, hi = (float(s[0]), float(s[1])) if isinstance(s, tuple) else (float(s), float(s))
        # ksize is piecewise increasing in sigma and drops at 3 and 5: its largest value is at hi or just below those
        worst = max(gaussian_ksize(x) for x in [hi] + [np.nextafter(b, 0.0) for b in (3.0, 5.0) if lo < b <= hi])
        if worst > MAX_BLUR_TAPS:
            raise GdrnError(f"COLOR_AUG_CODE: GaussianBlur(sigma={s!r}) needs a {worst}-tap kernel; at most "
                            f"{MAX_BLUR_TAPS} taps (sigma up to about 4.1) are supported")
    if name == "Invert" and (kw["min_value"] is not None or kw["max_value"] is not None):
        raise GdrnError("COLOR_AUG_CODE: Invert with min_value / max_value is not supported")
    if name == "AdditiveGaussianNoise" and (kw["loc"] != 0 or kw["per_channel"] is not True):
        raise GdrnError("COLOR_AUG_CODE: AdditiveGaussianNoise is supported with loc=0 and per_channel=True only")
    return {"kind": name, "prob": prob, **kw}


def parse_color_aug(code):
    """The imgaug program of INPUT.COLOR_AUG_CODE, parsed with ast (never evaluated):
    ``Sequential([Sometimes(p, Op(...)), ...], random_order=...)`` -> (ops, random_order).  Module prefixes
    (``iaa.``, ``pillike.``, ``iaa.contrast.``) are ignored; any other augmenter is rejected by name."""
    try:
        tree = ast.parse(code.strip(), mode="eval").body
    except SyntaxError as e:
        raise GdrnError(f"COLOR_AUG_CODE does not parse: {e}") from None
    if not isinstance(tree, ast.Call) or _call_name(tree) != "Sequential":
        raise GdrnError("COLOR_AUG_CODE: the program must be a Sequential([...])")
    if len(tree.args) != 1 or not isinstance(tree.args[0], ast.List):
        raise GdrnError("COLOR_AUG_CODE: Sequential takes one list of augmenters")
    random_order = False
    for k in tree.keywords:
        if k.arg != "random_order":
            raise GdrnError(f"COLOR_AUG_CODE: Sequential argument {k.arg!r} is not supported")
        random_order = bool(_literal(k.value, code))
    ops = [_parse_op(e, code) for e in tree.args[0].elts]
    if sum(op["kind"] == "CoarseDropout" for op in ops) > 1:
        raise GdrnError("COLOR_AUG_CODE: at most one CoarseDropout is supported (each image carries one cell mask)")
    return ops, random_order


def gaussian_ksize(sigma):
    """imgaug's _compute_gaussian_blur_ksize."""
    k = 3.3 * sigma if sigma < 3.0 else (2.9 * sigma if sigma < 5.0 else 2.6 * sigma)
    k = int(max(k, 5))
    return k + 1 if k % 2 == 0 else k


def gaussian_kernel_u8(sigma, n):
    """The 8-bit fixed-point kernel cv2.GaussianBlur uses for uint8 images: getGaussianKernelBitExact's
    exp(x^2 * -0.5 / sigma^2) weights (x on a step-2 grid scaled by 0.25), normalised, rounded to 1/256 with error
    diffusion from the outside in, and the centre taking the remainder so the taps sum to 256."""
    scale = -0.5 / (sigma * sigma) * 0.25
    half = (n - 1) // 2
    vals, s = [], 0.0
    for i in range(half):
        x = 1 - n + 2 * i
        t = math.exp((x * x) * scale)
        vals.append(t)
        s += t
    mul = 1.0 / (2.0 * s + 1.0)
    out = np.zeros(n, np.int32)
    err, tot = 0.0, 0
    for i in range(half):
        adj = vals[i] * mul * 256.0 + err
        v = int(np.rint(adj))
        err = adj - v
        out[i] = out[n - 1 - i] = v
        tot += v
    out[half] = 256 - 2 * tot
    return out


def _uniform(rng, spec, dtype=np.float32):
    if isinstance(spec, (tuple, list)):
        return dtype(rng.uniform(spec[0], spec[1]))
    return dtype(spec)


def _per_channel(rng, per_channel, draw):
    pc = 1.0 if per_channel is True else float(per_channel or 0)
    return [draw() for _ in range(3)] if (pc > 0 and rng.random() < pc) else [draw()] * 3


def _draw_op(rng, op, cell_hw):
    """-> (kind id or -1 when the op leaves the image unchanged, fpar [4], ipar [12], dropout cells or None)."""
    kind = op["kind"]
    f = np.zeros(N_FPAR, np.float32)
    i = np.zeros(N_IPAR, np.int32)
    cells = None
    if kind == "CoarseDropout":
        cells = (rng.random(cell_hw) >= float(_uniform(rng, op["p"], float))).astype(np.uint8)
    elif kind == "GaussianBlur":
        sigma = float(_uniform(rng, op["sigma"]))
        f[0] = sigma
        if sigma <= BLUR_EPS:
            return -1, f, i, None
        k = gaussian_ksize(sigma)
        i[0] = k
        i[1:1 + k] = gaussian_kernel_u8(sigma, k)
    elif kind.startswith("Enhance") or kind == "Grayscale":
        f[0] = _uniform(rng, op["factor" if kind.startswith("Enhance") else "alpha"])
    elif kind == "Add":
        v = op["value"]
        draw = (lambda: int(rng.integers(v[0], v[1] + 1))) if isinstance(v, (tuple, list)) else (lambda: int(v))
        i[:3] = _per_channel(rng, op["per_channel"], draw)
    elif kind == "Invert":
        i[:3] = _per_channel(rng, op["per_channel"], lambda: int(rng.random() < float(_uniform(rng, op["p"], float))))
    elif kind in ("Multiply", "LinearContrast"):
        key = "mul" if kind == "Multiply" else "alpha"
        f[:3] = _per_channel(rng, op["per_channel"], lambda: _uniform(rng, op[key]))
    elif kind == "AdditiveGaussianNoise":
        f[0] = _uniform(rng, op["scale"])
        i[:2] = rng.integers(0, 2 ** 32, 2, dtype=np.uint64).astype(np.uint32).view(np.int32)
    return COLOR_OPS[kind], f, i, cells


def dropout_grid(op, H, W):
    """The CoarseDropout cell grid: round(H * size_percent) x round(W * size_percent), at least min_size."""
    sp, mn = float(op["size_percent"]), int(op.get("min_size", 3))
    return max(int(round(H * sp)), mn), max(int(round(W * sp)), mn)


# --------------------------------------------------------------------------------------------- configuration
def train_resize_sizes(cfg):
    """The shortest-edge lengths build_gdrn_augmentation's training ResizeShortestEdge may pick: every
    MIN_SIZE_TRAIN entry ("choice"), or every integer of the [min, max] pair ("range").  Empty when
    INPUT.IMG_AUG_RESIZE is off."""
    if cfg_get(cfg, "INPUT.IMG_AUG_RESIZE", True) is False:
        return []
    short = cfg_get(cfg, "INPUT.MIN_SIZE_TRAIN", (480,))
    short = [int(v) for v in short] if isinstance(short, (list, tuple)) else [int(short)]
    if str(cfg_get(cfg, "INPUT.MIN_SIZE_TRAIN_SAMPLING", "choice")) == "range":
        if len(short) != 2:
            raise NotImplementedError(f"INPUT.MIN_SIZE_TRAIN={short} with MIN_SIZE_TRAIN_SAMPLING='range' needs (min, max)")
        short = list(range(short[0], short[1] + 1))
    return short


def check_train_config(cfg, im_size=None):
    """Reject, naming the setting, what the batcher does not build.  im_size (H, W): also require every training
    ResizeShortestEdge of MIN_SIZE_TRAIN / MAX_SIZE_TRAIN to be the identity for images of that size."""
    def bad(msg):
        raise NotImplementedError(msg)

    if cfg_get(cfg, "INPUT.WITH_DEPTH", False):
        bad("INPUT.WITH_DEPTH=True: depth inputs are not supported by the training batcher")
    sizes = train_resize_sizes(cfg)
    if im_size is not None:
        max_size = int(cfg_get(cfg, "INPUT.MAX_SIZE_TRAIN", 640))
        H, W = im_size
        for short in sizes:   # detectron2 leaves the image alone for a length of 0
            if short and _resize_shortest_edge_size(H, W, short, max_size) != (H, W):
                bad(f"INPUT.MIN_SIZE_TRAIN={cfg_get(cfg, 'INPUT.MIN_SIZE_TRAIN')} / INPUT.MAX_SIZE_TRAIN={max_size} "
                    f"resize the {W}x{H} training images (shortest edge {short}); only a ResizeShortestEdge that is the "
                    "identity for the split's image size is supported")
    dzi = str(cfg_get(cfg, "INPUT.DZI_TYPE", "uniform")).lower()
    if dzi not in ("uniform", "none"):
        bad(f"INPUT.DZI_TYPE={dzi!r}: only 'uniform' and 'none' are supported")
    if not cfg_get(cfg, "MODEL.POSE_NET.XYZ_ONLINE", False):
        bad("MODEL.POSE_NET.XYZ_ONLINE=False: the batcher renders xyz online only")
    if not cfg_get(cfg, "MODEL.POSE_NET.XYZ_BP", True):
        bad("MODEL.POSE_NET.XYZ_BP=False: only the back-projected online xyz is supported")
    xyz_loss = str(cfg_get(cfg, "MODEL.POSE_NET.LOSS_CFG.XYZ_LOSS_TYPE", "L1"))
    if "CE" in xyz_loss or "cls" in str(cfg_get(cfg, "MODEL.POSE_NET.NAME", "")):
        bad(f"MODEL.POSE_NET.LOSS_CFG.XYZ_LOSS_TYPE={xyz_loss!r}: CE xyz losses (roi_xyz_bin) are not supported")
    if str(cfg_get(cfg, "MODEL.POSE_NET.PNP_NET.COORD_2D_TYPE", "abs")) == "rel":
        bad('MODEL.POSE_NET.PNP_NET.COORD_2D_TYPE="rel" is not supported (only "abs")')
    if cfg_get(cfg, "TRAIN.VIS", False):
        bad("TRAIN.VIS=True is not supported (it also switches the mask crops to bilinear)")
    if str(cfg_get(cfg, "MODEL.BBOX_TYPE", "VISIB")).upper() not in ("AMODAL_CLIP", "VISIB"):
        bad(f"MODEL.BBOX_TYPE={cfg_get(cfg, 'MODEL.BBOX_TYPE')!r}: only AMODAL_CLIP and VISIB are supported")
    if cfg_get(cfg, "MODEL.BBOX_CROP_REAL", False) or cfg_get(cfg, "MODEL.BBOX_CROP_SYN", False):
        bad("MODEL.BBOX_CROP_REAL / BBOX_CROP_SYN are not supported")
    if str(cfg_get(cfg, "INPUT.FORMAT", "BGR")) != "BGR":
        bad(f"INPUT.FORMAT={cfg_get(cfg, 'INPUT.FORMAT')!r}: only BGR is supported")
    if str(cfg_get(cfg, "INPUT.BG_TYPE", "VOC_table")) not in ("VOC_table", "VOC", "coco"):
        bad(f"INPUT.BG_TYPE={cfg_get(cfg, 'INPUT.BG_TYPE')!r}: only VOC_table, VOC and coco are supported "
            "(SUN_RGBD needs background depth)")
    if not cfg_get(cfg, "INPUT.BG_KEEP_ASPECT_RATIO", True):
        bad("INPUT.BG_KEEP_ASPECT_RATIO=False is not supported")
    if float(cfg_get(cfg, "INPUT.COLOR_AUG_PROB", 0.0)) > 0:
        t = str(cfg_get(cfg, "INPUT.COLOR_AUG_TYPE", "ROI10D"))
        if t.lower() != "code":
            bad(f"INPUT.COLOR_AUG_TYPE={t!r}: only 'code' (an imgaug program) is supported")
        parse_color_aug(str(cfg_get(cfg, "INPUT.COLOR_AUG_CODE", "")))


# --------------------------------------------------------------------------------------------- the training split
# object names of the DATASETS.TRAIN entries <ds>_<obj>_train_*, where the name is not the object id itself
_NAMED_OBJS = {
    "lm": ["ape", "benchvise", "bowl", "camera", "can", "cat", "cup", "driller", "duck", "eggbox", "glue", "holepuncher",
           "iron", "lamp", "phone"],
    "ycbv": ["002_master_chef_can", "003_cracker_box", "004_sugar_box", "005_tomato_soup_can", "006_mustard_bottle",
             "007_tuna_fish_can", "008_pudding_box", "009_gelatin_box", "010_potted_meat_can", "011_banana",
             "019_pitcher_base", "021_bleach_cleanser", "024_bowl", "025_mug", "035_power_drill", "036_wood_block",
             "037_scissors", "040_large_marker", "051_large_clamp", "052_extra_large_clamp", "061_foam_brick"],
    "icbin": ["coffee_cup", "juice_carton"],
}
_NAMED_OBJS["lmo"] = _NAMED_OBJS["lm"]
TRAIN_DATASETS = ("lmo", "ycbv", "tless", "tudl", "icbin", "itodd", "hb")


def parse_train_name(name):
    """'<ds>[_<obj>]_train_pbr' or 'ycbv/tudl[_<obj>]_train_real' -> (dataset, obj token or None, split type)."""
    for st in ("pbr", "real"):
        suffix = "_train_" + st
        if name.endswith(suffix):
            head = name[: -len(suffix)]
            ds, _, obj = head.partition("_")
            if ds not in TRAIN_DATASETS or (st == "real" and ds not in ("ycbv", "tudl")):
                break
            return ds, (obj or None), st
    raise GdrnError(f"DATASETS.TRAIN entry {name!r} is not a supported BOP train split "
                    f"(<ds>[_<obj>]_train_pbr for {', '.join(TRAIN_DATASETS)}, ycbv/tudl[_<obj>]_train_real)")


def obj_id_of(ds, token):
    names = _NAMED_OBJS.get(ds)
    if names and token in names:
        return names.index(token) + 1
    head = token.split("_")[0]
    if head.isdigit() and (names is None or ds == "lmo"):
        return int(head)
    raise GdrnError(f"dataset {ds}: unknown object {token!r}")


def _bbox_center(K, t):
    proj = (K @ t.T).T
    return proj[:2] / proj[2]


class TrainSet:
    """The flattened training instances of the DATASETS.TRAIN splits, one sample per instance, filtered as the
    registrars and the train loader filter them: bbox_visib wider and taller than one pixel, a non-empty visible mask
    (scene_gt_info's px_count_visib, the mask_visib PNG's pixel count), visib_fract > DATALOADER.FILTER_VISIB_THR.
    Per object (label order): extents [m], roi_points (NUM_PM_POINTS model points: the first ones, shuffled once),
    sym_info (symmetry rotations or None) and fps points (fps{NUM_REGIONS}_and_center without the centre)."""

    def __init__(self, cfg, datasets_root, seed=0):
        """datasets_root: the reference's ``datasets/`` directory (BOP splits under BOP_DATASETS/)."""
        from . import bop_eval
        from .ply import load_ply

        names = cfg_get(cfg, "DATASETS.TRAIN", ())
        names = [names] if isinstance(names, str) else list(names)
        if not names:
            raise GdrnError("DATASETS.TRAIN is empty")
        parsed = [parse_train_name(n) for n in names]
        dss = {p[0] for p in parsed}
        if len(dss) != 1:
            raise GdrnError(f"DATASETS.TRAIN mixes datasets {sorted(dss)}; one dataset per batcher")
        self.dataset = ds = parsed[0][0]
        bop_root = os.path.join(datasets_root, "BOP_DATASETS")
        self.models_dir = models_path(bop_root, ds)
        info_path = os.path.join(self.models_dir, "models_info.json")
        if not os.path.exists(info_path):
            raise GdrnError(f"{info_path} does not exist")
        with open(info_path) as f:
            self.models_info = {int(k): v for k, v in json.load(f).items()}
        objs = {p[1] for p in parsed}
        if len(objs) != 1:
            raise GdrnError(f"DATASETS.TRAIN mixes object selections {sorted(map(str, objs))}")
        tok = parsed[0][1]
        self.obj_ids = [obj_id_of(ds, tok)] if tok else sorted(self.models_info)
        label_of = {o: i for i, o in enumerate(self.obj_ids)}
        thr = float(cfg_get(cfg, "DATALOADER.FILTER_VISIB_THR", 0.0))
        self.samples = []
        self.im_size = None
        for _, _, st in parsed:
            sp = split_params(bop_root, ds, "train", st)
            for scene_id, ims in plan_split(sp):
                sdir = os.path.join(sp["split_path"], "{:06d}".format(scene_id))
                gt_info = bop_eval.load_json(os.path.join(sdir, "scene_gt_info.json"), keys_to_int=True)
                for im in ims:
                    rgb = os.path.join(sdir, "rgb", "{:06d}{}".format(im["im_id"], sp["im_ext"]))
                    K = np.asarray(im["K"], np.float32).reshape(3, 3)
                    for k, gt in enumerate(im["gts"]):
                        o = int(gt["obj_id"])
                        if o not in label_of:
                            continue
                        info = gt_info[im["im_id"]][k]
                        if info["bbox_visib"][2] <= 1 or info["bbox_visib"][3] <= 1 or info.get("px_count_visib", 1) <= 0:
                            continue
                        if info.get("visib_fract", 1.0) <= thr:
                            continue
                        t = np.asarray(gt["cam_t_m2c"], np.float32).reshape(3) / 1000.0
                        self.samples.append({
                            "rgb": rgb,
                            "mask_visib": os.path.join(sdir, "mask_visib", "{:06d}_{:06d}.png".format(im["im_id"], k)),
                            "mask": os.path.join(sdir, "mask", "{:06d}_{:06d}.png".format(im["im_id"], k)),
                            "K": K, "R": np.asarray(gt["cam_R_m2c"], np.float32).reshape(3, 3), "t": t,
                            "label": label_of[o], "bbox_obj": list(info["bbox_obj"]), "bbox_visib": list(info["bbox_visib"]),
                            "centroid": _bbox_center(K, t),
                        })
        if not self.samples:
            raise GdrnError(f"DATASETS.TRAIN {names}: no training instances after filtering")
        # per object
        rng = np.random.default_rng([seed, 1])
        num_pm = int(cfg_get(cfg, "MODEL.POSE_NET.LOSS_CFG.NUM_PM_POINTS", 3000))
        pts = [load_ply(os.path.join(self.models_dir, "obj_{:06d}.ply".format(o)), vertex_scale=0.001)["pts"]
               for o in self.obj_ids]
        self.extents = np.array([p.max(0) - p.min(0) for p in pts], np.float32)
        num = min(min(p.shape[0] for p in pts), num_pm)
        self.roi_points = np.stack([p[rng.permutation(num)] for p in pts]).astype(np.float32)
        self.sym_info = []
        for o in self.obj_ids:
            mi = self.models_info[o]
            if "symmetries_discrete" in mi or "symmetries_continuous" in mi:
                syms = bop_eval.get_symmetry_transformations(mi, max_sym_disc_step=0.01)
                self.sym_info.append(np.array([s["R"] for s in syms], dtype=np.float32))
            else:
                self.sym_info.append(None)
        self.num_regions = int(cfg_get(cfg, "MODEL.POSE_NET.GEO_HEAD.NUM_REGIONS", 64))
        self.fps_points = None
        if self.num_regions > 1:
            fps_path = os.path.join(self.models_dir, "fps_points.pkl")
            if not os.path.exists(fps_path):
                raise GdrnError(f"{fps_path} does not exist: write it with `python -m gdrnpp_bop2022_b200.train_batch "
                                f"compute_fps --dataset {ds}`")
            with open(fps_path, "rb") as f:
                fps = pickle.load(f)
            key = f"fps{self.num_regions}_and_center"
            self.fps_points = np.stack([np.asarray(fps[str(o)][key], np.float32)[:-1] for o in self.obj_ids])
        self.model_paths = [os.path.join(self.models_dir, "obj_{:06d}.ply".format(o)) for o in self.obj_ids]

    def __len__(self):
        return len(self.samples)


def background_paths(cfg, datasets_root, rng):
    """_bg_img_paths (base_data_loader.py:339-411) for BG_TYPE VOC_table / VOC / coco, listed in sorted order; then
    NUM_BG_IMGS of them drawn with replacement."""
    bg_type = str(cfg_get(cfg, "INPUT.BG_TYPE", "VOC_table"))
    root = resolve_path(str(cfg_get(cfg, "INPUT.BG_IMGS_ROOT", "datasets/VOCdevkit/VOC2012/")), datasets_root)
    if not os.path.isdir(root):
        raise GdrnError(f"INPUT.BG_IMGS_ROOT {root} does not exist")
    if bg_type == "coco":
        paths = [os.path.join(root, f) for f in sorted(os.listdir(root)) if ".png" in f or "jpg" in f]
    elif bg_type == "VOC_table":
        with open(os.path.join(root, "ImageSets/Main/diningtable_trainval.txt")) as f:
            ids = [ln.split()[0] for ln in f.read().splitlines() if ln.strip() and ln.split()[1] == "1"]
        paths = [os.path.join(root, "JPEGImages/{}.jpg".format(i)) for i in ids]
    elif bg_type == "VOC":
        d = os.path.join(root, "JPEGImages")
        paths = [os.path.join(d, f) for f in sorted(os.listdir(d)) if ".jpg" in f]
    else:
        raise NotImplementedError(f"INPUT.BG_TYPE={bg_type!r} is not supported")
    if not paths:
        raise GdrnError(f"INPUT.BG_IMGS_ROOT {root}: no background images")
    num = min(len(paths), int(cfg_get(cfg, "INPUT.NUM_BG_IMGS", 10000)))
    return [paths[i] for i in rng.choice(len(paths), num)]


# --------------------------------------------------------------------------------------------- per-sample records
class Sampler:
    """Draws the per-sample records of a batch (everything random in read_data_train) from one Generator."""

    def __init__(self, cfg, n_samples, n_bg, im_hw):
        self.n_samples, self.n_bg = n_samples, n_bg
        self.H, self.W = im_hw
        self.change_bg = float(cfg_get(cfg, "INPUT.CHANGE_BG_PROB", 0.0))
        self.truncate_fg = bool(cfg_get(cfg, "INPUT.TRUNCATE_FG", False))
        self.color_prob = float(cfg_get(cfg, "INPUT.COLOR_AUG_PROB", 0.0))
        self.ops, self.random_order = ([], False)
        if self.color_prob > 0:
            self.ops, self.random_order = parse_color_aug(str(cfg_get(cfg, "INPUT.COLOR_AUG_CODE", "")))
        self.S = max(len(self.ops), 1)
        drop = [op for op in self.ops if op["kind"] == "CoarseDropout"]
        self.cell_hw = dropout_grid(drop[0], self.H, self.W) if drop else (1, 1)   # parse_color_aug allows one
        self.dzi = str(cfg_get(cfg, "INPUT.DZI_TYPE", "uniform")).lower()
        self.dzi_scale = float(cfg_get(cfg, "INPUT.DZI_SCALE_RATIO", 0.25))
        self.dzi_shift = float(cfg_get(cfg, "INPUT.DZI_SHIFT_RATIO", 0.25))

    def draw(self, rng, n):
        """-> record dict of arrays with a leading sample axis n."""
        S, (ch, cw) = self.S, self.cell_hw
        r = {"index": np.zeros(n, np.int64), "do_bg": np.zeros(n, np.int32), "bg_index": np.zeros(n, np.int64),
             "trunc_side": np.full(n, 4, np.int32), "trunc_u": np.zeros(n, np.float64),
             "do_color": np.zeros(n, np.int32), "perm": np.tile(np.arange(S, dtype=np.int32), (n, 1)),
             "op_on": np.zeros((n, S), np.int32), "kind_at": np.full((n, S), -1, np.int32),
             "fpar": np.zeros((n, S, N_FPAR), np.float32), "ipar": np.zeros((n, S, N_IPAR), np.int32),
             "cells": np.ones((n, ch, cw), np.uint8), "dzi_scale": np.ones(n, np.float64),
             "dzi_shift": np.zeros((n, 2), np.float64)}
        for b in range(n):
            r["index"][b] = rng.integers(self.n_samples)
            if rng.random() < self.change_bg:
                r["do_bg"][b] = 1
                r["bg_index"][b] = rng.integers(self.n_bg)
                if self.truncate_fg:
                    rnd = rng.random()
                    r["trunc_side"][b] = min(int(rnd / 0.2), 4)
                    r["trunc_u"][b] = rng.random()
            if self.ops and rng.random() < self.color_prob:
                r["do_color"][b] = 1
                perm = rng.permutation(len(self.ops)).astype(np.int32) if self.random_order else np.arange(len(self.ops))
                r["perm"][b, :len(self.ops)] = perm
                for c, op in enumerate(self.ops):
                    if rng.random() < op["prob"]:
                        r["op_on"][b, c] = 1
                        kind, f, i, cells = _draw_op(rng, op, self.cell_hw)
                        s = int(np.nonzero(perm == c)[0][0])
                        r["kind_at"][b, s], r["fpar"][b, s], r["ipar"][b, s] = kind, f, i
                        if cells is not None:
                            r["cells"][b] = cells
            if self.dzi == "uniform":
                r["dzi_scale"][b] = 1 + self.dzi_scale * (2 * rng.random() - 1)
                r["dzi_shift"][b] = self.dzi_shift * (2 * rng.random(2) - 1)
        return r


def take(rec, sel):
    return {k: v[sel] for k, v in rec.items()}


def put(rec, sel, sub):
    for k, v in sub.items():
        rec[k][sel] = v


def roi_geometry(cfg, ts, rec):
    """Per-sample box arithmetic of read_data_train in float64: the BBOX_TYPE box, aug_bbox_DZI's centre and scale,
    roi_wh, resize_ratio and trans_ratio.  -> dict of arrays."""
    H, W = ts.im_size
    out_res = int(cfg_get(cfg, "MODEL.POSE_NET.OUTPUT_RES", 64))
    pad = float(cfg_get(cfg, "INPUT.DZI_PAD_SCALE", 1.0))
    amodal = str(cfg_get(cfg, "MODEL.BBOX_TYPE", "VISIB")).upper() == "AMODAL_CLIP"
    dzi = str(cfg_get(cfg, "INPUT.DZI_TYPE", "uniform")).lower()
    n = len(rec["index"])
    g = {"center": np.zeros((n, 2)), "scale": np.zeros(n), "wh": np.zeros((n, 2)), "trans_ratio": np.zeros((n, 3))}
    for b in range(n):
        s = ts.samples[rec["index"][b]]
        if amodal:
            x, y, w, h = s["bbox_obj"]
            x1, y1, x2, y2 = max(float(x), 0.0), max(float(y), 0.0), min(float(x + w), float(W)), min(float(y + h), float(H))
        else:
            x, y, w, h = s["bbox_visib"]
            x1, y1 = min(max(float(x), 0.0), float(W)), min(max(float(y), 0.0), float(H))
            x2, y2 = min(max(float(x + w), 0.0), float(W)), min(max(float(y + h), 0.0), float(H))
        cx, cy, bw, bh = 0.5 * (x1 + x2), 0.5 * (y1 + y2), x2 - x1, y2 - y1
        if dzi == "uniform":
            center = np.array([cx + bw * rec["dzi_shift"][b, 0], cy + bh * rec["dzi_shift"][b, 1]])
            scale = max(y2 - y1, x2 - x1) * rec["dzi_scale"][b] * pad
        else:
            center = np.array([cx, cy])
            scale = max(y2 - y1, x2 - x1)
        scale = min(scale, max(H, W)) * 1.0
        bw, bh = max(bw, 1), max(bh, 1)
        resize_ratio = out_res / scale
        delta = s["centroid"] - center
        g["center"][b], g["scale"][b], g["wh"][b] = center, scale, (bw, bh)
        # float64, as the reference's numpy-scalar box makes it (a python-float scale would round t_z / ratio to f32)
        g["trans_ratio"][b] = (delta[0] / bw, delta[1] / bh, float(s["t"][2]) / resize_ratio)
    return g


def bg_layout(bg_hw, H, W):
    """get_bg_image's top-left crop and resize_short_edge's size for a bg_h x bg_w background on an H x W image
    (base_data_loader.py:480-551, data_utils.py:208-235) -> (crop_h, crop_w, resized_h, resized_w, 1 / fx)."""
    bg_h, bg_w = bg_hw
    ratio = float(H) / float(W)
    crop_h, crop_w = bg_h, bg_w
    same = (H / W < 1 and bg_h / bg_w < 1) or (H / W >= 1 and bg_h / bg_w >= 1)
    if bg_h >= bg_w:
        h_new = int(np.ceil(bg_w * ratio))
        if not same or h_new < bg_h:
            crop_h = h_new
    else:
        w_new = int(np.ceil(bg_h / ratio))
        if not same or w_new < bg_w:
            crop_w = w_new
    crop_h, crop_w = min(crop_h, bg_h), min(crop_w, bg_w)
    target, max_size = min(H, W), max(H, W)
    s_min, s_max = min(crop_h, crop_w), max(crop_h, crop_w)
    scale = float(target) / float(s_min)
    if np.round(scale * s_max) > max_size:
        scale = float(max_size) / float(s_max)
    rh, rw = int(np.rint(crop_h * scale)), int(np.rint(crop_w * scale))
    if rh > H or rw > W:
        raise GdrnError(f"background of {bg_w}x{bg_h} resizes to {rw}x{rh}, larger than the {W}x{H} image")
    return crop_h, crop_w, rh, rw, 1.0 / scale


def read_mask(path):
    import cv2

    m = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if m is None:
        raise GdrnError(f"cannot read mask {path}")
    return (m.reshape(m.shape[0], m.shape[1], -1)[..., 0] > 0).astype(np.uint8)


def read_bgr(path):
    im = read_image(path)
    return np.repeat(im, 3, axis=2) if im.shape[2] == 1 else im


def decode(ts, bg_paths, rec):
    """Host decode of one (sub-)batch: images [n,H,W,3], mask_visib / mask_full [n,H,W] u8 0/1, and the backgrounds
    of the samples that replace theirs."""
    n = len(rec["index"])
    H, W = ts.im_size
    imgs = np.empty((n, H, W, 3), np.uint8)
    mv = np.empty((n, H, W), np.uint8)
    mf = np.empty((n, H, W), np.uint8)
    bgs = [None] * n
    for b in range(n):
        s = ts.samples[rec["index"][b]]
        im = read_bgr(s["rgb"])
        if im.shape[:2] != (H, W):
            raise GdrnError(f"{s['rgb']} is {im.shape[1]}x{im.shape[0]}, expected {W}x{H}")
        imgs[b], mv[b], mf[b] = im, read_mask(s["mask_visib"]), read_mask(s["mask"])
        if rec["do_bg"][b]:
            bgs[b] = read_bgr(bg_paths[rec["bg_index"][b]])
    return imgs, mv, mf, bgs


# --------------------------------------------------------------------------------------------- device pipeline
def build_images(cfg, ts, rec, dec, dev, stats=None, staging=None):
    """Composite + colour steps + ROI crops of one (sub-)batch on `dev` -> dict of device tensors incl. 'counts'.
    staging: a dict of pinned host buffers reused across calls; the caller synchronises (the pixel-count copy) before
    the next call, so no upload from an earlier call is still reading them."""
    import torch

    L = _lib.lib()
    H, W = ts.im_size
    imgs, mv, mf, bgs = dec
    n = imgs.shape[0]
    in_res = int(cfg_get(cfg, "MODEL.POSE_NET.INPUT_RES", 256))
    out_res = int(cfg_get(cfg, "MODEL.POSE_NET.OUTPUT_RES", 64))
    st = _lib.current_stream()

    def up(a):
        a = np.ascontiguousarray(a)
        if staging is None:
            return torch.from_numpy(a).to(dev)
        key = len(staging.setdefault("_order", []))
        staging["_order"].append(key)
        buf = staging.get(key)
        if buf is None or buf.numel() < a.nbytes:
            buf = staging[key] = torch.empty(max(a.nbytes, 1), dtype=torch.uint8, pin_memory=True)
        buf[:a.nbytes].numpy()[...] = a.reshape(-1).view(np.uint8)
        return buf[:a.nbytes].to(dev, non_blocking=True).view(torch.from_numpy(a[:0]).dtype).view(a.shape)

    def ev(name):
        if stats is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            stats.setdefault("events", []).append((name, e))

    ev("upload")
    im_a, mv_d, mf_d = up(imgs), up(mv), up(mf)
    meta = np.zeros((n, 7), np.int32)
    bscale = np.ones((n, 2), np.float64)
    off = np.zeros(n, np.int64)
    pool, pos = [], 0
    for b in range(n):
        if bgs[b] is None:
            continue
        ch_, cw_, rh, rw, inv = bg_layout(bgs[b].shape[:2], H, W)
        meta[b] = (1, bgs[b].shape[0], bgs[b].shape[1], ch_, cw_, rh, rw)
        bscale[b] = inv
        off[b] = pos
        pool.append(bgs[b].reshape(-1))
        pos += bgs[b].size
    pool_d = up(np.concatenate(pool)) if pool else torch.zeros(1, dtype=torch.uint8, device=dev)
    bbox = torch.tensor([H, -1, W, -1], dtype=torch.int32).repeat(n, 1).to(dev)
    keep = torch.empty((n, 4), dtype=torch.int32, device=dev)
    side = np.where(rec["do_bg"] > 0, rec["trunc_side"], 4).astype(np.int32)
    meta_d, bscale_d, off_d, side_d, u_d = up(meta), up(bscale), up(off), up(side), up(rec["trunc_u"])
    ev("composite")
    _lib.check(L.gdrn_train_composite(_lib.ptr(im_a), _lib.ptr(mv_d), n, H, W, _lib.ptr(pool_d), _lib.ptr(off_d),
                                      _lib.ptr(meta_d), _lib.ptr(bscale_d), _lib.ptr(side_d), _lib.ptr(u_d), _lib.ptr(bbox),
                                      _lib.ptr(keep), st), "gdrn_train_composite")
    S = rec["kind_at"].shape[1]
    kind_at = np.where(rec["do_color"][:, None] > 0, rec["kind_at"], -1).astype(np.int32)
    if (kind_at >= 0).any():
        ev("color")
        ch, cw = rec["cells"].shape[1:]
        kind_d, fpar_d, ipar_d, cells_d = up(kind_at), up(rec["fpar"]), up(rec["ipar"]), up(rec["cells"])
        sums = torch.zeros(n, dtype=torch.int64, device=dev)
        im_b = torch.empty_like(im_a)
        for s in range(S):
            if (kind_at[:, s] < 0).all():
                continue
            if (kind_at[:, s] == COLOR_OPS["EnhanceContrast"]).any():
                _lib.check(L.gdrn_train_luma_sum(_lib.ptr(im_a), n, H, W, _lib.ptr(kind_d), S, s, _lib.ptr(sums), st),
                           "gdrn_train_luma_sum")
            _lib.check(L.gdrn_train_color_step(_lib.ptr(im_a), _lib.ptr(im_b), n, H, W, _lib.ptr(kind_d), _lib.ptr(fpar_d),
                                               _lib.ptr(ipar_d), S, s, _lib.ptr(cells_d), ch, cw, _lib.ptr(sums), st),
                       "gdrn_train_color_step")
            im_a, im_b = im_b, im_a
    geo = roi_geometry(cfg, ts, rec)
    cs = np.concatenate([geo["center"], geo["scale"][:, None]], axis=1)
    mean = np.asarray(cfg_get(cfg, "MODEL.PIXEL_MEAN", [0.0, 0.0, 0.0]), np.float64)
    std = np.asarray(cfg_get(cfg, "MODEL.PIXEL_STD", [255.0, 255.0, 255.0]), np.float64)
    out = {"roi_img": torch.empty((n, 3, in_res, in_res), dtype=torch.float32, device=dev),
           "roi_coord_2d": torch.empty((n, 2, out_res, out_res), dtype=torch.float32, device=dev),
           "roi_mask_trunc": torch.empty((n, out_res, out_res), dtype=torch.float32, device=dev),
           "roi_mask_visib": torch.empty((n, out_res, out_res), dtype=torch.float32, device=dev),
           "roi_mask_full": torch.empty((n, out_res, out_res), dtype=torch.float32, device=dev),
           "counts": torch.empty((n, 2), dtype=torch.int32, device=dev)}
    ev("crop")
    cs_d = up(cs)
    _lib.check(L.gdrn_train_roi_crop(_lib.ptr(im_a), _lib.ptr(mv_d), _lib.ptr(mf_d), _lib.ptr(keep), _lib.ptr(cs_d), n, H, W,
                                     in_res, out_res, mean.ctypes.data_as(_lib.c_void_p), std.ctypes.data_as(_lib.c_void_p),
                                     _lib.ptr(out["roi_img"]), _lib.ptr(out["roi_coord_2d"]), _lib.ptr(out["roi_mask_trunc"]),
                                     _lib.ptr(out["roi_mask_visib"]), _lib.ptr(out["roi_mask_full"]), _lib.ptr(out["counts"]),
                                     st), "gdrn_train_roi_crop")
    ev("end")
    out["geo"] = geo
    out["image"] = im_a   # the augmented images (tests compare them with the oracle)
    return out


MIN_ROI_PIXELS = 32   # data_loader_online.py:543


class GdrnTrainBatcher:
    """Iterator over training batches: each a dict with the keys, dtypes and shapes batch_data_train_online returns for
    the config (roi_img [B,3,in,in], roi_cls, roi_coord_2d, roi_cam, roi_center, roi_scale, resize_ratio, roi_zoom_K,
    roi_wh, roi_extent, roi_trans_ratio, roi_mask_trunc / visib / full, ego_rot, trans, roi_points, sym_info (list),
    roi_mask_obj, roi_fps_points and roi_region (NUM_REGIONS > 1), roi_xyz).  Batch k draws its records from
    numpy.random.default_rng([seed, 1000 + k]); the records of the last batch are kept in ``last_records`` and its
    augmented images [B,H,W,3] u8 (device) in ``last_images``."""

    def __init__(self, cfg, datasets_root, *, seed=0, batch_size=None, device="cuda", num_workers=8):
        import torch

        check_train_config(cfg)
        self.cfg, self.seed = cfg, int(seed)
        self.batch_size = int(batch_size or cfg_get(cfg, "SOLVER.IMS_PER_BATCH", 32))
        self.device = torch.device(device)
        self.ts = TrainSet(cfg, datasets_root, seed=seed)
        H, W = read_bgr(self.ts.samples[0]["rgb"]).shape[:2]
        check_train_config(cfg, (H, W))
        self.ts.im_size = (H, W)
        change_bg = float(cfg_get(cfg, "INPUT.CHANGE_BG_PROB", 0.0)) > 0
        self.bg_paths = background_paths(cfg, datasets_root, np.random.default_rng([seed, 2])) if change_bg else []
        self.sampler = Sampler(cfg, len(self.ts), max(len(self.bg_paths), 1), (H, W))
        from .renderer import load_models

        self.models = load_models(self.ts.model_paths, scale_to_meter=0.001, device=self.device)
        self.pool = ThreadPoolExecutor(max(1, num_workers))
        self.k = 0
        self.pending = None
        self.last_records = None
        self.last_images = None
        self.stats = None   # a dict here collects the stage events of the next batch (bench_train_batch.py)
        self.staging = {}

    def _decode_async(self, rec):
        n = len(rec["index"])
        parts = max(1, min(n, self.pool._max_workers))
        chunks = np.array_split(np.arange(n), parts)
        futs = [self.pool.submit(decode, self.ts, self.bg_paths, take(rec, c)) for c in chunks]
        return futs

    @staticmethod
    def _join(futs):
        parts = [f.result() for f in futs]
        return (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]),
                np.concatenate([p[2] for p in parts]), [bg for p in parts for bg in p[3]])

    def _draw(self, k):
        rng = np.random.default_rng([self.seed, 1000 + k])
        rec = self.sampler.draw(rng, self.batch_size)
        return rng, rec, self._decode_async(rec)

    def __iter__(self):
        return self

    def __next__(self):
        import torch

        if self.pending is None:
            self.pending = self._draw(self.k)
        rng, rec, futs = self.pending
        dec = self._join(futs)
        self.k += 1
        self.pending = self._draw(self.k)   # the next batch decodes while this one runs on the GPU
        with torch.cuda.device(self.device):
            self.staging["_order"] = []
            out = build_images(self.cfg, self.ts, rec, dec, self.device, self.stats, self.staging)
            for _ in range(1000):
                bad = (out["counts"].cpu().numpy() < MIN_ROI_PIXELS).any(axis=1)
                if not bad.any():
                    break
                sel = np.nonzero(bad)[0]
                sub = self.sampler.draw(rng, len(sel))
                put(rec, sel, sub)
                redo = build_images(self.cfg, self.ts, sub, decode(self.ts, self.bg_paths, sub), self.device)
                idx = torch.as_tensor(sel, device=self.device)
                for key in ("roi_img", "roi_coord_2d", "roi_mask_trunc", "roi_mask_visib", "roi_mask_full", "counts",
                            "image"):
                    out[key][idx] = redo[key]
                for key in out["geo"]:
                    out["geo"][key][sel] = redo["geo"][key]
            else:
                raise GdrnError("no sample with at least 32 cropped mask pixels after 1000 redraws")
            self.last_records = rec
            self.last_images = out["image"]
            return self._assemble(rec, out)

    def _assemble(self, rec, out):
        import torch

        from .online_targets import render_roi_targets
        from .renderer import get_K_crop_resize

        dev, ts, cfg = self.device, self.ts, self.cfg
        if self.stats is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.stats["events"].append(("targets", e))
        out_res = int(cfg_get(cfg, "MODEL.POSE_NET.OUTPUT_RES", 64))
        samples = [ts.samples[i] for i in rec["index"]]
        labels = np.array([s["label"] for s in samples])
        geo = out["geo"]
        f32 = dict(dtype=torch.float32, device=dev)
        bs = len(samples)
        batch = {"roi_img": out["roi_img"], "roi_cls": torch.as_tensor(labels, dtype=torch.long, device=dev),
                 "roi_coord_2d": out["roi_coord_2d"],
                 "roi_cam": torch.as_tensor(np.stack([s["K"] for s in samples]), **f32),
                 "roi_center": torch.as_tensor(geo["center"].astype(np.float32), **f32),
                 "roi_scale": torch.as_tensor(geo["scale"], **f32),
                 "resize_ratio": torch.as_tensor(out_res / geo["scale"], **f32)}
        crop_xy = batch["roi_center"] - batch["roi_scale"].view(bs, -1) / 2
        batch["roi_zoom_K"] = get_K_crop_resize(batch["roi_cam"], crop_xy, out_res / batch["roi_scale"].view(bs, -1))
        batch["roi_wh"] = torch.as_tensor(geo["wh"].astype(np.float32), **f32)
        batch["roi_extent"] = torch.as_tensor(ts.extents[labels], **f32)
        batch["roi_trans_ratio"] = torch.as_tensor(geo["trans_ratio"].astype(np.float32), **f32)
        for key in ("roi_mask_trunc", "roi_mask_visib", "roi_mask_full"):
            batch[key] = out[key]
        batch["ego_rot"] = torch.as_tensor(np.stack([s["R"] for s in samples]), **f32)
        batch["trans"] = torch.as_tensor(np.stack([s["t"] for s in samples]), **f32)
        batch["roi_points"] = torch.as_tensor(ts.roi_points[labels], **f32)
        batch["sym_info"] = [ts.sym_info[lab] for lab in labels]
        fps = torch.as_tensor(ts.fps_points[labels], **f32) if ts.fps_points is not None else None
        tg = render_roi_targets(self.models, batch["roi_cls"], batch["ego_rot"], batch["trans"], batch["roi_zoom_K"],
                                batch["roi_extent"], fps, out_res=out_res)
        batch["roi_mask_obj"] = tg["roi_mask_obj"]
        batch["roi_mask_trunc"] = batch["roi_mask_trunc"] * batch["roi_mask_obj"]
        batch["roi_mask_visib"] = batch["roi_mask_visib"] * batch["roi_mask_obj"]
        if fps is not None:
            batch["roi_fps_points"] = fps
            batch["roi_region"] = tg["roi_region"]
        batch["roi_xyz"] = tg["roi_xyz"]
        if self.stats is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.stats["events"].append(("done", e))
        return batch

    def close(self):
        self.pool.shutdown(wait=True)


# --------------------------------------------------------------------------------------------- fps_points.pkl
FPS_COUNTS = (4, 8, 12, 16, 20, 32, 64, 128, 256)


def compute_fps(models_dir, obj_ids=None):
    """<ds>_1_compute_fps.py: {str(obj_id): {f"fps{n}_and_center": [n + 1, 3]}} with the model points in metres,
    native_ops.farthest_point_sampling(init_center=True) and the points' mean as the last row."""
    from .native_ops import farthest_point_sampling
    from .ply import load_ply

    if obj_ids is None:
        with open(os.path.join(models_dir, "models_info.json")) as f:
            obj_ids = sorted(int(k) for k in json.load(f))
    out = {}
    for o in obj_ids:
        pts = load_ply(os.path.join(models_dir, "obj_{:06d}.ply".format(o)), vertex_scale=0.001)["pts"].astype(np.float32)
        center = np.array([[np.average(pts[:, 0]), np.average(pts[:, 1]), np.average(pts[:, 2])]])
        out[str(o)] = {f"fps{n}_and_center": np.concatenate([farthest_point_sampling(pts, n, init_center=True), center], 0)
                       for n in FPS_COUNTS}
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m gdrnpp_bop2022_b200.train_batch")
    sub = ap.add_subparsers(dest="cmd", required=True)
    p = sub.add_parser("compute_fps", help="write <models>/fps_points.pkl of a BOP dataset")
    p.add_argument("--dataset", required=True)
    p.add_argument("--datasets-root", default="datasets", help="the directory holding BOP_DATASETS/")
    p.add_argument("--models-dir", default=None)
    a = ap.parse_args(argv)
    d = models_path(os.path.join(a.datasets_root, "BOP_DATASETS"), a.dataset, a.models_dir)
    res = compute_fps(d)
    path = os.path.join(d, "fps_points.pkl")
    with open(path, "wb") as f:
        pickle.dump(res, f)
    print(f"wrote {path} ({len(res)} objects)")


if __name__ == "__main__":
    main()
