"""YOLOX-X (depth 1.33, width 1.25, 8 classes, 640 x 640) multi-scale test-time augmentation with the scales of the
shipped BOP test configs (1, 0.75, 0.83, 1.12, 1.25: network inputs 640, 480, 544, 736 and 800, 43 428 anchors):
per-call latency and images/s of YOLOX.forward(augment=True) on the CUDA kernels (B = 1 replayed as a captured CUDA
graph, B = 8 eager) in both precisions, the plain forward at the same batch for the ratio, and yolox_post.postprocess
(conf 0.001, nms 0.65, class-aware, as yolox_inference_on_dataset runs it) on the TTA output with the number of
candidates that pass the threshold.  Beside them, the oracle's functional forward (F.interpolate + the network per scale)
in torch eager with cuDNN, in fp32 with TF32 off and in fp16 like the reference's half_test=True.  Weights are synthetic
(gdrnpp_bop2022_b200.synthetic.make_yolox_state_dict).  Prints one JSON line per row, with the card name and power limit.

  python bench_yolox_tta.py [--min-window-ms 1000] [--batches 1,8]

Each number is the median of three timed windows of at least --min-window-ms each, with the min and max beside it.
"""
import argparse
import json
from types import SimpleNamespace

import torch

from bench_yolox import card, timed

SCALES = (1, 0.75, 0.83, 1.12, 1.25)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-window-ms", type=float, default=1000.0, help="each timed window lasts at least this long")
    ap.add_argument("--batches", default="1,8")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_yolox_tta.py needs a GPU"
    from gdrnpp_bop2022_b200.synthetic import make_yolox_state_dict
    from gdrnpp_bop2022_b200.yolox_model import YOLOX
    from gdrnpp_bop2022_b200.yolox_post import postprocess_padded
    from oracle.yolox_oracle import yolox_forward
    from oracle.yolox_tta_oracle import yolox_forward_tta

    name = card()
    dev = torch.device("cuda")
    sd = make_yolox_state_dict(yolox_forward, 1.33, 1.25, 8, seed=0, device="cuda")
    batches = [int(b) for b in args.batches.split(",")]
    cfg = SimpleNamespace(scales=SCALES)
    rows = []

    def run(fn):
        fn()
        torch.cuda.synchronize()
        t = timed(fn, 3, warmup=1, repeats=1)[0]   # rough per-call time: size the windows to min_window_ms
        return timed(fn, max(5, int(args.min_window_ms / max(t, 1e-3)) + 1))

    def report(impl, precision, B, stats, **extra):
        ms, lo, hi = stats
        r = {"impl": impl, "precision": precision, "batch": B, "ms_per_call": round(ms, 3),
             "ms_min_max": [round(lo, 3), round(hi, 3)], "images_per_s": round(1000.0 * B / ms, 1), **extra, "card": name}
        rows.append(r)
        print(json.dumps(r), flush=True)
        return ms

    for precision in ("bf16x3", "bf16"):
        m = YOLOX(1.33, 1.25, 8, max_batch=max(batches), precision=precision).eval()
        m.load_state_dict(sd)
        m.to(dev)
        for B in batches:
            x = torch.rand((B, 3, 640, 640), device=dev) * 255
            graph = B == 1
            if graph:
                replay_tta, out = m.capture_graph(x, augment=True, cfg=cfg)
                replay_plain, _ = m.capture_graph(x)
                t_tta, t_plain = run(replay_tta), run(replay_plain)
                det = out["det_preds"]
            else:
                t_tta, t_plain = run(lambda: m(x, augment=True, cfg=cfg)), run(lambda: m(x))
                det = m(x, augment=True, cfg=cfg)["det_preds"]
            sfx = " (graph)" if graph else ""
            ms = report("cuda_kernels tta" + sfx, precision, B, t_tta, anchors=det.shape[1])
            report("cuda_kernels plain" + sfx, precision, B, t_plain, anchors=m._engines[(640, 640)].A,
                   tta_over_plain=round(ms / t_plain[0], 3))
            cand = int(((det[..., 4] * det[..., 5:].max(-1).values) >= 0.001).sum().item())
            report("yolox_postprocess", precision, B, run(lambda: postprocess_padded(det, 8, 0.001, 0.65)),
                   candidates_per_image=round(cand / B, 1))
            del det
        del m
        torch.cuda.empty_cache()

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    for dtype, label in ((torch.float32, "fp32"), (torch.float16, "fp16")):
        sdt = {k: (v.to(dev, dtype) if v.is_floating_point() else v) for k, v in sd.items()}
        for B in batches:
            x = (torch.rand((B, 3, 640, 640), device=dev) * 255).to(dtype)
            with torch.no_grad():
                report("torch_eager_cudnn tta", label, B, run(lambda: yolox_forward_tta(sdt, x, 1.33, 8, SCALES)))
        del sdt
        torch.cuda.empty_cache()
    print(json.dumps({"summary": rows, "card": name}))


if __name__ == "__main__":
    main()
