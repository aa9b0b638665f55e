#!/usr/bin/env python
"""UFRCNN+ train-step timing on one GPU, with the card's name, power limit and max SM clock read in the same run: forward, losses, one
batched host sync, backward and Adam at batch 2 x 128^3 (lidc_exp 3D config), CUDA events after a warm-up.  Prints one JSON line; --out FILE
also writes it there.

  python tools/ufrcnn_bench.py [--steps 20] [--warmup 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from medicaldetectiontoolkit_b200 import ufrcnn  # noqa: E402
from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


def time_events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ufrcnn_bench: needs a CUDA device")
    cf = make_cf('ufrcnn', 3, (128, 128, 128))
    torch.manual_seed(0)
    net = ufrcnn.net(cf).cuda()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    batch = synthetic_batch(cf, 2, seed=0)

    def step():
        r = net.train_forward(batch)
        opt.zero_grad(set_to_none=True)
        r['torch_loss'].backward()
        opt.step()

    ms = time_events(step, a.steps, a.warmup)
    res = {"card": card(), "train_step_ms": round(ms, 2), "patches_per_s": round(2 * 1000 / ms, 2), "batch": 2, "patch": [128, 128, 128],
           "post_nms_rois_training": cf.post_nms_rois_training, "steps": a.steps, "warmup": a.warmup}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
