"""Training-batch throughput: GdrnTrainBatcher (GPU) against the NumPy / cv2 / PIL restatement of read_data_train run
by 8 worker processes, the shape of the reference's DataLoader with DATALOADER.NUM_WORKERS = 8.

Synthetic BOP PBR scenes (640x480 JPEGs, masks, box meshes) and VOC-style backgrounds are generated from a seed in a
temporary directory; the config is the shipped AugCosyAAEGray one (CHANGE_BG_PROB 0.5, TRUNCATE_FG, COLOR_AUG_PROB 0.8
with the 13-op imgaug program, DZI uniform, 64 regions).  Prints one JSON line: batches/s and samples/s of both paths,
the mean time of each GPU stage from CUDA events, and the card's name and power limit read in the same run."""
import argparse
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time
from multiprocessing import get_context

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return name, power
    except Exception as e:   # the numbers are still printed, marked with why the card is unknown
        return f"unknown ({e})", "unknown"


_W = {}


def _init_worker(cfg, datasets_root, bg_paths, im_size, seed):
    from gdrnpp_bop2022_b200 import train_batch as TB

    ts = TB.TrainSet(cfg, datasets_root, seed=seed)
    ts.im_size = im_size
    _W.update(cfg=cfg, ts=ts, bg=bg_paths)


def _oracle_sample(rec):
    from oracle import train_batch_oracle as O

    return O.replay(_W["cfg"], _W["ts"], _W["bg"], rec)["counts"]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=48)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-batches", type=int, default=2)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--images", type=int, default=60)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)

    import torch

    from gdrnpp_bop2022_b200 import train_batch as TB
    from gdrnpp_bop2022_b200.synthetic import shipped_train_cfg, write_bop_train_tree

    if not torch.cuda.is_available():
        raise SystemExit("bench_train_batch.py needs a CUDA device")
    name, power = _gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        base = write_bop_train_tree(tmp, num_images=a.images, num_scenes=3, insts_per_image=6, seed=a.seed, num_bg=24)
        datasets_root = tmp
        fps = TB.compute_fps(os.path.join(base, "models"))
        with open(os.path.join(base, "models", "fps_points.pkl"), "wb") as f:
            pickle.dump(fps, f)
        cfg = shipped_train_cfg()
        bt = TB.GdrnTrainBatcher(cfg, datasets_root, seed=a.seed, batch_size=a.batch, num_workers=a.workers)
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
        # the oracle path: per-sample replay on a process pool
        recs = [bt.sampler.draw(np.random.default_rng([a.seed, 50 + k]), a.batch) for k in range(a.oracle_batches)]
        singles = [TB.take(r, [i]) for r in recs for i in range(a.batch)]
        ctx = get_context("spawn")
        with ctx.Pool(a.workers, initializer=_init_worker,
                      initargs=(cfg, datasets_root, bt.bg_paths, bt.ts.im_size, a.seed)) as pool:
            pool.map(_oracle_sample, singles[: a.workers])   # workers up
            t0 = time.perf_counter()
            pool.map(_oracle_sample, singles, chunksize=1)
            cpu_s = (time.perf_counter() - t0) / a.oracle_batches
        bt.close()
    print(json.dumps({
        "workload": f"GDRN training batches, B={a.batch}, 640x480, shipped AugCosyAAEGray config",
        "gpu": name, "power_limit": power,
        "gpu_batches_per_s": round(1.0 / gpu_s, 3), "gpu_samples_per_s": round(a.batch / gpu_s, 1),
        "oracle_workers": a.workers, "oracle_batches_per_s": round(1.0 / cpu_s, 3),
        "oracle_samples_per_s": round(a.batch / cpu_s, 1),
        "gpu_stage_ms": {k: round(float(np.mean(v)), 3) for k, v in stages.items()},
    }))


if __name__ == "__main__":
    main()
