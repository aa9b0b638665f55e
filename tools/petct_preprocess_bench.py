#!/usr/bin/env python
"""Cost of the PET-CT preprocessing (petct_preprocessing.py, csrc/petct_preprocess.cu) for one synthetic patient.  Prints one JSON line per
measurement, the first naming the card, its power limit and its maximum SM clock.  The patient: a 512 x 512 x 300 int16 CT at (0.7, 0.7,
2.0) mm with two lungs in a body over 200 slices, a 200 x 200 x 300 float32 PET at 4 mm and a 4-D stack of two segments on the CT's grid.

- `resample_ct_ms`: the CT onto the new (0.976562, 0.976562, 3.27) grid (367 x 367 x 183); `resample_pet_ms`: the PET onto that grid;
- `components_ms`: the per-slice body components of the resampled CT; `criterion_ms`: one get_z_crops criterion launch;
- `normalize_ms`: the two-channel normalisation of the cropped slab;
  each the median device time from CUDA events over repeated calls on device-resident inputs after a warm-up;
- `patient_s`: the whole process_patient from host arrays (uploads, kernels, downloads), a host clock around a call that ends in a copy
  to the host; the file writes and reading are excluded;
- `numpy_resample_ct_s`, `numpy_zcrop_s`: oracle/petct_preprocess_oracle.py (numpy / scipy, fp64) for the CT resample and for the
  reference's get_z_crops on the resampled CT, on one host core.

    python tools/petct_preprocess_bench.py [--reps 20] [--no-numpy]"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import petct_preprocess_oracle as PO  # noqa: E402
from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import petct_preprocessing as P  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def make_patient():
    Z, Y, X = 300, 512, 512
    y, x = np.ogrid[:Y, :X]
    body = ((y - 256) / 200.0) ** 2 + ((x - 256) / 220.0) ** 2 <= 1
    lungs = (((y - 250) / 120.0) ** 2 + ((x - 150) / 70.0) ** 2 <= 1) | (((y - 250) / 120.0) ** 2 + ((x - 362) / 70.0) ** 2 <= 1)
    plane = np.where(body, 40, -1000).astype(np.int16)
    ct = np.broadcast_to(plane, (Z, Y, X)).copy()
    ct[50:250][:, lungs] = -850
    ct += np.random.RandomState(0).randint(-30, 30, (1, Y, X)).astype(np.int16)
    ct_geom = ((0.7, 0.7, 2.0), (-179.0, -179.0, -300.0), P.IDENTITY)
    pet = np.random.RandomState(1).gamma(2.0, 0.5, (300, 200, 200)).astype(np.float32)
    pet_geom = ((4.0, 4.0, 4.0), (-400.0, -400.0, -600.0), P.IDENTITY)
    rd = np.zeros((2, X, Y, Z), np.uint8, order='F')
    rd[0, 200:230, 220:250, 100:110] = 1
    rd[1, 300:320, 260:280, 150:160] = 1
    header = {'space directions': np.array([[np.nan] * 3, [0.7, 0, 0], [0, 0.7, 0], [0, 0, 2.0]]), 'space origin': np.array([-179.0, -179.0, -300.0]),
              'Segment0_Name': 'T_primary', 'Segment1_Name': 'N_inflammation'}
    return ct, ct_geom, pet, pet_geom, rd, header


def device_ms(fn, reps):
    for _ in range(2):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-numpy", action="store_true")
    a = ap.parse_args()
    emit(card=card())
    ops = P.CudaOps()
    ct, ct_geom, pet, pet_geom, rd, header = make_patient()
    g_ct = P.Grid.of(ct.shape, *ct_geom)
    g_new = P.new_ct_grid(g_ct)
    g_pet = P.Grid.of(pet.shape, *pet_geom)
    ct_d, pet_d = ops.upload(ct), ops.upload(pet)
    x = ops.resample(ct_d, g_ct, g_new, np.int16)
    p = ops.resample(pet_d, g_pet, g_new, np.float32)
    emit(measure="resample_ct_ms", shape=list(g_new.shape), value=round(device_ms(lambda: ops.resample(ct_d, g_ct, g_new, np.int16), a.reps), 3))
    emit(measure="resample_pet_ms", value=round(device_ms(lambda: ops.resample(pet_d, g_pet, g_new, np.float32), a.reps), 3))
    _, first, stats = ops.body_components(x)
    emit(measure="components_ms", value=round(device_ms(lambda: ops.body_components(x), a.reps), 3))
    flags = torch.empty(g_new.shape[0], dtype=torch.uint8, device=x.device)
    Z, Y, X = g_new.shape
    crit = lambda: L.check(L.load().mdt_petct_zcrop_criterion(L.ptr(first), L.ptr(stats), Z, Y, X, 1500, 2, 20000.0, L.ptr(flags),
                                                              L.stream_ptr()))
    emit(measure="criterion_ms", value=round(device_ms(crit, a.reps), 3))
    zmin, zmax = P.get_z_crops(x, 0, ops=ops)
    lo, hi = P._slab(zmin, zmax, Z)
    emit(measure="zcrop", z_min=int(zmin), z_max=int(zmax))
    emit(measure="normalize_ms", slices=hi - lo, value=round(device_ms(lambda: ops.normalize(x[lo:hi], p[lo:hi]), a.reps), 3))
    runs = []
    for _ in range(3):
        torch.cuda.synchronize()
        t = time.perf_counter()
        P.process_patient(ct, ct_geom, pet, pet_geom, rd, header, ops=ops)
        runs.append(time.perf_counter() - t)
    emit(measure="patient_s", value=round(float(np.median(runs)), 3), runs=[round(r, 3) for r in runs])
    if not a.no_numpy:
        t = time.perf_counter()
        xi = PO.resample(ct, g_ct.as_dict(), g_new.as_dict(), np.int16)
        emit(measure="numpy_resample_ct_s", value=round(time.perf_counter() - t, 2), equal_to_device=bool(np.array_equal(xi, x.cpu().numpy())))
        t = time.perf_counter()
        want = PO.get_z_crops(xi, 0)
        emit(measure="numpy_zcrop_s", value=round(time.perf_counter() - t, 2), equal_to_device=[int(v) for v in want] == [int(zmin), int(zmax)])


if __name__ == "__main__":
    main()
