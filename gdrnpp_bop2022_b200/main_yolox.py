"""Command line of the reference's detector test script (test_yolox.sh -> main_yolox.py --eval-only):

    python -m gdrnpp_bop2022_b200.main_yolox --config-file CFG --eval-only --datasets_root DATASETS \\
        train.init_checkpoint=CKPT [test.augment=False ...] [--det_file PATH]

Overrides take the LazyConfig ``key=value`` form.  ``--datasets_root`` is the reference's ``datasets/`` directory
(BOP_DATASETS/<name>/... below it).  Results go to ``<train.output_dir>/inference/<DATASETS.TEST>/``; the detection file
of the pose loop (DATASETS.DET_FILES_TEST of main_gdrn) to ``--det_file``, by default
``<output dir>/test_bboxes/<config name>.json``.
"""
import argparse
import ast
import os
import sys

_OVERRIDABLE = {"train.init_checkpoint", "train.output_dir", "test.augment", "test.scales", "test.conf_thr", "test.nms_thr",
                "test.test_size", "test.half_test", "test.amp_test", "test.test_dataset_names", "DATASETS.TEST",
                "val.eval_cached"}


def _parse_value(v):
    try:
        return ast.literal_eval(v)
    except (ValueError, SyntaxError):
        return v


def apply_overrides(cfg, opts):
    """LazyConfig key=value overrides -> (cfg updated in place, init_checkpoint or None)."""
    ckpt = None
    for tok in opts:
        k, sep, v = tok.partition("=")
        if not sep:
            raise SystemExit(f"{tok!r} is not key=value")
        if k not in _OVERRIDABLE:
            raise SystemExit(f"override {k!r} is not supported (one of {sorted(_OVERRIDABLE)})")
        val = _parse_value(v)
        if k == "train.init_checkpoint":
            ckpt = v
        elif k == "train.output_dir":
            cfg.output_dir = v
        elif k in ("test.test_dataset_names", "DATASETS.TEST"):
            cfg.test_dataset_names = tuple(val) if isinstance(val, (list, tuple)) else (val,)
        elif k == "val.eval_cached":
            cfg.eval_cached = bool(val)
        else:
            name = k.split(".", 1)[1]
            setattr(cfg, name, tuple(val) if isinstance(val, list) else val)
    return cfg, ckpt


def parse_args(argv=None):
    """Options may come before or after the key=value overrides (test_yolox.sh passes the overrides last)."""
    ap = argparse.ArgumentParser(description="YOLOX dataset test loop on the GPU (main_yolox.py --eval-only)")
    ap.add_argument("--config-file", required=True)
    ap.add_argument("--eval-only", action="store_true", help="accepted for compatibility; only evaluation is supported")
    ap.add_argument("--datasets_root", default="datasets")
    ap.add_argument("--det_file", default=None, help="path of the converted detection file for the pose loop")
    ap.add_argument("--max_batch", type=int, default=8, help="images per forward")
    ap.add_argument("--precision", default=None, choices=(None, "bf16x3", "bf16"))
    ap.add_argument("--num-gpus", "--num_gpus", type=int, default=1)
    ap.add_argument("opts", nargs="*", default=[], help="LazyConfig key=value overrides")
    return ap.parse_intermixed_args(argv)


def main(argv=None):
    args = parse_args(argv)
    if args.num_gpus != 1:
        raise SystemExit("--num-gpus: the test loop runs on one GPU")
    import torch

    from . import yolox_evaluator as YE
    from .yolox_model import YOLOX, load_yolox_config

    cfg = load_yolox_config(args.config_file)
    cfg, ckpt = apply_overrides(cfg, args.opts)
    YE.check_test_config(cfg)
    if not ckpt:
        raise SystemExit("train.init_checkpoint is not set (train.init_checkpoint=CKPT)")
    precision = YE.precision_of(cfg, args.precision)
    model = YOLOX(cfg.depth, cfg.width, cfg.num_classes, max_batch=args.max_batch, precision=precision).eval()
    ck = torch.load(ckpt, map_location="cpu")
    sd = ck.get("model", ck)
    model.load_state_dict({k[len("_module."):] if k.startswith("_module.") else k: v for k, v in sd.items()})
    model.to("cuda")
    name = cfg.test_dataset_names[0]
    ts = YE.YoloxTestSet(name, args.datasets_root)
    records = YE.yolox_inference_on_dataset(cfg, model, args.datasets_root, max_batch=args.max_batch, test_set=ts)
    out_dir = os.path.join(cfg.output_dir, "inference", name)
    config_name = os.path.splitext(os.path.basename(args.config_file))[0]
    res = YE.YoloxDatasetEvaluator(cfg, ts, out_dir, args.det_file, config_name).evaluate(records)
    print("wrote", res["files"]["det_file"])
    return res


if __name__ == "__main__":
    main(sys.argv[1:])
