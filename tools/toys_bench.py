#!/usr/bin/env python
"""Cost of the toy-experiment generator (generate_toys.py, csrc/toys.cu).  Prints one JSON line per measurement, the first naming the card
and its power limit:

- `launch_ms` for 256 and 1024 images: device time of one mdt_toy_images launch from CUDA events after a warm-up (median of --reps), and
  the rate of its output writes (1.64 MB per image) in GB/s;
- `experiment`: generate_experiment('donuts_shape', 1500, 1000) into a temporary directory (about 4.1 GB of .npy files): `total_s`, a
  host clock around the call; `device_d2h_s`, the same launches and copies into the pinned buffer without the file writes, timed on
  their own; `writes_s` = total_s - device_d2h_s, derived, not timed as such (the call overlaps the next launch with the writes);
- `oracle_ms_per_image`: oracle/toys_oracle.py (numpy, one host thread) per image.

    python tools/toys_bench.py [--reps 10] [--out-dir DIR]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import toys_oracle as TO  # noqa: E402
from medicaldetectiontoolkit_b200 import generate_toys as G  # noqa: E402

IMG_BYTES = 2 * 320 * 320 * 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def launch_ms(n, reps):
    ops = G.CudaOps()
    keys = np.array([[0, 0, i] for i in range(n)], dtype=np.uint32)
    for _ in range(2):
        ops.images(keys, 'donuts_shape', (20, 20), 10)
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.images(keys, 'donuts_shape', (20, 20), 10)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def device_d2h_s(n_images):
    ops = G.CudaOps()
    host = ops.staging(G.CHUNK)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c0 in range(0, n_images, G.CHUNK):
        m = min(G.CHUNK, n_images - c0)
        img, params = ops.images(np.array([[0, 0, i] for i in range(c0, c0 + m)], dtype=np.uint32), 'donuts_shape', (20, 20), 10)
        host[:m].copy_(img)
        params.cpu()
    return time.perf_counter() - t0


def main():
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--reps", type=int, default=10)
    p.add_argument("--out-dir", default=None, help="where the experiment is written (default: a temporary directory, removed after)")
    a = p.parse_args()
    emit(card=card(), torch=torch.__version__)
    for n in (256, 1024):
        ms = launch_ms(n, a.reps)
        emit(kind="launch", images=n, launch_ms=round(ms, 3), write_gbs=round(n * IMG_BYTES / ms / 1e6, 1))
    n_train, n_test = 1500, 1000
    tmp = tempfile.mkdtemp(dir=a.out_dir)
    try:
        free = shutil.disk_usage(tmp).free
        if free < 2 * (n_train + n_test) * IMG_BYTES:
            emit(kind="experiment", skipped="%.1f GB free in %s" % (free / 1e9, tmp))
        else:
            t0 = time.perf_counter()
            G.generate_experiment(tmp, 'donuts_shape', n_train, n_test, 'donuts_shape', seed=0)
            total = time.perf_counter() - t0
            dev = device_d2h_s(n_train + n_test)
            emit(kind="experiment", images=n_train + n_test, total_s=round(total, 2), device_d2h_s=round(dev, 2), writes_s=round(total - dev, 2),
                 gb_written=round((n_train + n_test) * IMG_BYTES / 1e9, 2))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    t0 = time.perf_counter()
    for i in range(20):
        TO.image([0, 0, i], 'donuts_shape', (20, 20))
    emit(kind="oracle", oracle_ms_per_image=round((time.perf_counter() - t0) / 20 * 1e3, 2))


if __name__ == "__main__":
    main()
