#!/usr/bin/env python
"""Cost of the data loader (data_loader.py, csrc/loader.cu) per batch.  Prints one JSON line per measurement, the first naming the card and
its power limit.  Synthetic lidc-sized patients (512 x 512 x 250, float32 image, uint8 seg with a few lesions) are written to a temporary
directory first.  Every time is a host clock around the call and a device synchronise, so it includes the host's share (random draws,
memory-mapped reads, staging copies, table building):

- `lidc3d`: a lidc 3D BatchGenerator batch (8 x 156x156x96), `first_touch` with the foreground index built for every patient in the batch,
  `cached` once every patient is indexed;
- `lidc2d`: a lidc 2D batch (20 x 300^2), cached;
- `patient3d`: one PatientBatchIterator patient (3D, 128x128x64 patches, batch returned as host arrays);
- `numpy`: the same with the numpy stand-in for the device ops (tests/_loader_cases.NumpyOps) on one core, rebuilding the foreground
  index for every element as the reference's np.unique / np.argwhere scan the whole patient for every element.

    python tools/loader_bench.py [--iters 5] [--patients 4]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _loader_cases as LC  # noqa: E402
from medicaldetectiontoolkit_b200 import data_loader as D  # noqa: E402
from medicaldetectiontoolkit_b200.configs import make_cf  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def write_patients(path, n, seed=0):
    import pandas as pd
    rs = np.random.RandomState(seed)
    rows = []
    for i in range(n):
        Z, Y, X = 250, 512, 512
        seg = np.zeros((Z, Y, X), np.uint8)
        k = int(rs.randint(1, 5))
        for j in range(k):
            z, y, x = rs.randint(10, Z - 20), rs.randint(40, Y - 60), rs.randint(40, X - 60)
            seg[z:z + rs.randint(3, 12), y:y + rs.randint(5, 30), x:x + rs.randint(5, 30)] = j + 1
        np.save(os.path.join(path, 'b%d_img.npy' % i), rs.randn(Z, Y, X).astype(np.float32))
        np.save(os.path.join(path, 'b%d_rois.npy' % i), seg)
        rows.append({'pid': 'b%d' % i, 'class_target': [int(rs.randint(1, 6)) for _ in range(k)],
                     'fg_slices': [int(z) for z in np.nonzero(seg.reshape(Z, -1).any(1))[0]]})
    pd.DataFrame(rows).to_pickle(os.path.join(path, 'info_df.pickle'))


def timed(fn, sync=True):
    t = time.perf_counter()
    out = fn()
    if sync:
        torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--patients", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loader_bench needs a CUDA device")
    emit(card=card(), torch=torch.__version__)
    with tempfile.TemporaryDirectory() as tmp:
        write_patients(tmp, a.patients)
        data = LC.dataset('lidc', tmp)
        cf3 = make_cf('retina_unet', 3, (128, 128, 64), exp='lidc_exp', batch_size=8)
        cf2 = make_cf('mrcnn', 2, (288, 288), exp='lidc_exp', batch_size=20)
        cf3.head_classes = cf2.head_classes = 2           # np.random.choice over the patients: the synthetic targets need no balancing
        # first touch: a fresh generator (empty index cache) per batch
        first = []
        for i in range(a.iters):
            gen = D.BatchGenerator(data, 8, cf3, seed=i, rank=0)
            first.append(timed(gen.generate_train_batch)[0])
        gen = D.BatchGenerator(data, 8, cf3, seed=0, rank=0)
        for pid, p in data.items():
            gen.fg_index(pid, np.load(p['seg'], mmap_mode='r'))
        gen.generate_train_batch()
        cached = [timed(gen.generate_train_batch)[0] for _ in range(a.iters)]
        emit(case='lidc3d', batch='8 x 156x156x96', first_touch_ms=1e3 * float(np.median(first)), cached_ms=1e3 * float(np.median(cached)),
             cached_min_ms=1e3 * min(cached))
        gen2 = D.BatchGenerator(data, 20, cf2, seed=0, rank=0)
        for pid, p in data.items():
            gen2.fg_index(pid, np.load(p['seg'], mmap_mode='r'))
        gen2.generate_train_batch()
        t2 = [timed(gen2.generate_train_batch)[0] for _ in range(a.iters)]
        emit(case='lidc2d', batch='20 x 300x300', cached_ms=1e3 * float(np.median(t2)), cached_min_ms=1e3 * min(t2))
        it = D.PatientBatchIterator(data, cf3)
        it.generate_train_batch()
        tp, b = [], None
        for _ in range(a.iters):
            t, b = timed(it.generate_train_batch)
            tp.append(t)
        emit(case='patient3d', patches=int(b['data'].shape[0]), patch='128x128x64', ms=1e3 * float(np.median(tp)))
        # numpy stand-in on one core, the index rebuilt for every element
        torch.set_num_threads(1)
        ops = LC.NumpyOps()
        gn = D.BatchGenerator(data, 8, cf3, seed=0, rank=0, ops=ops)
        gn2 = D.BatchGenerator(data, 20, cf2, seed=0, rank=0, ops=ops)
        for g in (gn, gn2):
            g.fg_index = (lambda g, build: lambda pid, seg: (g._index.clear(), build(pid, seg))[1])(g, g.fg_index)
        n3 = [timed(gn.generate_train_batch, sync=False)[0] for _ in range(2)]
        n2 = timed(gn2.generate_train_batch, sync=False)[0]
        itn = D.PatientBatchIterator(data, cf3, ops=ops)
        npat = timed(itn.generate_train_batch, sync=False)[0]
        emit(case='numpy', cores=1, lidc3d_ms=1e3 * float(np.median(n3)), lidc2d_ms=1e3 * n2, patient3d_ms=1e3 * npat)


if __name__ == "__main__":
    main()
