"""One parity-mode forward at a small batch (default B = 5, the per-image case of BASELINE configs[4]) repeated N times, for
a CUDA-event timing of the graph replay.  Usage: python tools/fwd_small.py [B] [reps]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gdrnpp_bop2022_b200.gdrn_model import GDRN_DoubleMask, default_cfg  # noqa: E402
from gdrnpp_bop2022_b200.synthetic import make_batch, make_state_dict  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 5
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
dev = torch.device("cuda:0")
model = GDRN_DoubleMask(default_cfg(), max_batch=max(B, 2), precision="bf16x3")
model.load_state_dict(make_state_dict())
model.to(dev)
keys = ("roi_img", "roi_classes", "roi_coord_2d", "roi_cams", "roi_centers", "roi_whs", "resize_ratios", "roi_extents")
b = {k: v.to(dev) for k, v in make_batch(B=B, seed=3).items() if k in keys}
kw = {k: b[k] for k in keys if k != "roi_img"}
for _ in range(reps):
    model(b["roi_img"], **kw)
torch.cuda.synchronize()
if os.environ.get("FWD_SMALL_GRAPH", "1") != "0":
    replay, out = model.capture_graph(b)
    for _ in range(3):
        replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        replay()
    e1.record()
    torch.cuda.synchronize()
    print("B=%d graph replay: %.3f ms per forward (%.0f ROIs/s)" % (B, e0.elapsed_time(e1) / 50, B * 50 / e0.elapsed_time(e1) * 1e3))
