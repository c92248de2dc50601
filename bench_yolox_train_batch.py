"""YOLOX training-batch throughput: YoloxTrainBatcher (GPU) against the NumPy / cv2 restatement of
MosaicDetection.__getitem__ run by 4 worker processes, the shape of the reference's loader (dataloader.train.num_workers
= 4 per GPU).

A synthetic LM-O PBR split (640x480 JPEGs) is generated from a seed in a temporary directory; the config is the shipped
yolox_x_640_augCozyAAEhsv_ranger_30_epochs_lmo_pbr_lmo_bop_test one (mosaic and mixup always on, the wrapper's HSV pass,
COLOR_AUG_PROB 0.8 with the 12-op imgaug program).  Both paths include the JPEG decode.  Prints one JSON line: batches/s
and samples/s of both paths, the mean time of each GPU stage from CUDA events, and the card's name and power limit read
in the same run."""
import argparse
import json
import os
import sys
import tempfile
import time
from multiprocessing import get_context

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_train_batch import _gpu_info  # noqa: E402

_W = {}


def _init_worker(cfg, datasets_root):
    from gdrnpp_bop2022_b200 import yolox_train_batch as YT

    _W.update(cfg=cfg, ts=YT.YoloxTrainSet(cfg, datasets_root))


def _oracle_sample(rec):
    from gdrnpp_bop2022_b200 import yolox_train_batch as YT
    from oracle import yolox_train_batch_oracle as O

    ts = _W["ts"]
    return O.replay(rec, YT.decode(ts, rec, [0]), lambda i: ts.images[i]["labels"],
                    source_format=_W["cfg"].aug_wrapper["FORMAT"])[1]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-batches", type=int, default=2)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--images", type=int, default=60)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)

    import torch

    from gdrnpp_bop2022_b200 import yolox_train_batch as YT
    from gdrnpp_bop2022_b200.synthetic import write_bop_train_tree, write_yolox_train_config
    from gdrnpp_bop2022_b200.yolox_model import load_yolox_config

    if not torch.cuda.is_available():
        raise SystemExit("bench_yolox_train_batch.py needs a CUDA device")
    name, power = _gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        write_bop_train_tree(tmp, dataset="lmo", num_images=a.images, num_scenes=3, insts_per_image=6, seed=a.seed,
                             obj_ids=(1, 5, 6, 8, 9, 10, 11, 12), num_bg=1)
        cfg = load_yolox_config(write_yolox_train_config(os.path.join(tmp, "configs")))
        bt = YT.YoloxTrainBatcher(cfg, tmp, seed=a.seed, batch_size=a.batch)
        for _ in range(a.warmup):
            next(bt)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            next(bt)
            torch.cuda.synchronize()
        gpu_s = (time.perf_counter() - t0) / a.steps
        # stage times from CUDA events, in a run of their own
        stages = {}
        for _ in range(max(3, a.steps // 4)):
            bt.stats = {}
            next(bt)
            torch.cuda.synchronize()
            ev = bt.stats["events"]
            for (n0, e0), (_, e1) in zip(ev[:-1], ev[1:]):
                stages.setdefault(n0, []).append(e0.elapsed_time(e1))
        bt.stats = None
        recs = [bt.sampler.draw(np.random.default_rng([a.seed, 50 + k]), a.batch) for k in range(a.oracle_batches)]
        singles = [{k: v[i:i + 1] for k, v in r.items()} for r in recs for i in range(a.batch)]
        with get_context("spawn").Pool(a.workers, initializer=_init_worker, initargs=(cfg, tmp)) as pool:
            pool.map(_oracle_sample, singles[: a.workers])   # workers up
            t0 = time.perf_counter()
            pool.map(_oracle_sample, singles, chunksize=1)
            cpu_s = (time.perf_counter() - t0) / a.oracle_batches
        bt.close()
    print(json.dumps({
        "workload": f"YOLOX training batches, B={a.batch}, 640x480 -> 640x640, shipped lmo_pbr config",
        "gpu": name, "power_limit": power,
        "gpu_batches_per_s": round(1.0 / gpu_s, 3), "gpu_samples_per_s": round(a.batch / gpu_s, 1),
        "oracle_workers": a.workers, "oracle_batches_per_s": round(1.0 / cpu_s, 3),
        "oracle_samples_per_s": round(a.batch / cpu_s, 1),
        "gpu_stage_ms": {k: round(float(np.mean(v)), 3) for k, v in stages.items()},
    }))


if __name__ == "__main__":
    main()
