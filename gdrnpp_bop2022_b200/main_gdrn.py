"""Command line of the reference's test scripts (test_gdrn.sh / test_gdrn_depth_refine.sh -> main_gdrn.py --eval-only):

    python -m gdrnpp_bop2022_b200.main_gdrn --config-file CFG --eval-only --datasets_root DATASETS \\
        --opts MODEL.WEIGHTS=CKPT [KEY=VALUE ...]

``--datasets_root`` is the reference's ``datasets/`` directory (BOP_DATASETS/<name>/... below it); paths in
DATASETS.DET_FILES_TEST that start with ``datasets/`` are resolved against it.  Per-object (class-agnostic) checkpoints:
``MODEL.WEIGHTS=<obj_id>=<ckpt> <obj_id>=<ckpt> ...`` runs every object's network in one pass; a single per-object
checkpoint names its object with ``--obj_ids``.

``--opts TEST.SAVE_RESULTS_ONLY=True`` runs the reference's save_gdrn.sh instead: gdrn_save_result_of_dataset writes
results.pkl (per ROI the pose and the visible / amodal masks as COCO RLE) to
``<OUTPUT_DIR>/inference_<model name>/<DATASETS.TEST[0]>`` (or ``--output_dir``), with exactly one DATASETS.TEST
entry.  Per-object checkpoints given together write one results.pkl under ``inference_per_object/`` (the reference
runs one process per object).
"""
import argparse
import ast
import os
import re
import sys

from .gdrn_model import _NS, load_py_config


def _parse_value(v):
    try:
        return ast.literal_eval(v)
    except (ValueError, SyntaxError):
        return v


def set_opt(cfg, key, value):
    cur = cfg
    parts = key.split(".")
    for p in parts[:-1]:
        nxt = getattr(cur, p, None)
        if nxt is None:
            nxt = _NS()
            setattr(cur, p, nxt)
        cur = nxt
    setattr(cur, parts[-1], value)


def parse_opts(opts):
    """KEY=VALUE pairs -> ({key: value}, per-object weights {obj_id: path} or None)."""
    out, per_obj, last = {}, {}, None
    for tok in opts:
        k, sep, v = tok.partition("=")
        if not sep:
            raise SystemExit(f"--opts: {tok!r} is not KEY=VALUE")
        if re.fullmatch(r"\d+", k) and last == "MODEL.WEIGHTS":
            per_obj[int(k)] = v
            continue
        if k == "MODEL.WEIGHTS" and re.match(r"\d+=", v):
            ok, _, ov = v.partition("=")
            per_obj[int(ok)] = ov
        else:
            out[k] = _parse_value(v) if k != "MODEL.WEIGHTS" else v
        last = k
    return out, (per_obj or None)


def main(argv=None):
    ap = argparse.ArgumentParser(description="GDRNPP dataset test loop on the GPU (main_gdrn.py --eval-only)")
    ap.add_argument("--config-file", required=True)
    ap.add_argument("--eval-only", action="store_true", help="accepted for compatibility; only evaluation is supported")
    ap.add_argument("--datasets_root", default="datasets")
    ap.add_argument("--output_dir", default=None, help="default: <OUTPUT_DIR>/inference/<VAL.DATASET_NAME>")
    ap.add_argument("--obj_ids", default=None, help="comma-separated obj_ids a per-object checkpoint covers")
    ap.add_argument("--max_batch", type=int, default=64, help="ROIs per forward (whole images)")
    ap.add_argument("--precision", default=None, choices=(None, "bf16x3", "bf16"))
    ap.add_argument("--num_gpus", type=int, default=1)
    ap.add_argument("--opts", nargs=argparse.REMAINDER, default=[])
    args = ap.parse_args(argv)
    if args.num_gpus != 1:
        raise SystemExit("--num_gpus: the test loop runs on one GPU")
    from . import gdrn_evaluator as G

    cfg = load_py_config(args.config_file)
    opts, per_obj = parse_opts(args.opts)
    for k, v in opts.items():
        set_opt(cfg, k, v)
    G.check_config(cfg)
    weights = per_obj or G.cfg_get(cfg, "MODEL.WEIGHTS")
    if not weights:
        raise SystemExit("MODEL.WEIGHTS is not set (--opts MODEL.WEIGHTS=CKPT)")
    train_obj_ids = [int(x) for x in args.obj_ids.split(",")] if args.obj_ids else (sorted(per_obj) if per_obj else None)
    save_only = bool(G.cfg_get(cfg, "TEST.SAVE_RESULTS_ONLY", False))
    if save_only:
        try:
            save_dir = G.save_results_dir(cfg, per_object=bool(per_obj))
        except ValueError as e:
            raise SystemExit(str(e))
        save_dir = args.output_dir or save_dir
    ts = G.TestSet(cfg, args.datasets_root, train_obj_ids)
    model = G.build_model(cfg, weights, obj_ids=ts.obj_ids, precision=args.precision, max_batch=args.max_batch)
    if save_only:
        G.gdrn_save_result_of_dataset(cfg, model, args.datasets_root, save_dir, train_obj_ids=train_obj_ids,
                                      max_batch=args.max_batch, test_set=ts)
        path = os.path.join(save_dir, "results.pkl")
        print("wrote", path)
        return {"results": path}
    records = G.gdrn_inference_on_dataset(cfg, model, args.datasets_root, train_obj_ids=train_obj_ids,
                                          max_batch=args.max_batch, test_set=ts)
    out_dir = args.output_dir or os.path.join(str(G.cfg_get(cfg, "OUTPUT_DIR", "output")), "inference",
                                              str(G.cfg_get(cfg, "VAL.DATASET_NAME")))
    res = G.GdrnDatasetEvaluator(cfg, args.datasets_root, out_dir, G.exp_id(cfg, args.config_file)).evaluate(records)
    print("wrote", res["csv"])
    return res


if __name__ == "__main__":
    main(sys.argv[1:])
