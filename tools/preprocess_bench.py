#!/usr/bin/env python
"""Cost of the LIDC preprocessing (preprocessing.py, csrc/preprocess.cu) per patient.  Prints one JSON line per measurement, the first
naming the card and its power limit.  Synthetic patients from a seed, each with 3 ROIs x 4 raters of small blobs:

- `up_z`: 512 x 512 x 250 int16 at spacing (0.65, 0.65, 2.5): x and y blurred and downsampled, z upsampled;
- `down`: 512 x 512 x 400 int16 at spacing (0.55, 0.55, 1.0): every axis blurred and downsampled.

Per kind:
- `ct_ms`, `roi_ms`: device time of one CT resample + normalisation, and of one ROI (4 rater resamples + the vote), from CUDA events over
  repeated calls on device-resident sources after a warm-up (median);
- `patient_s`: the whole pp_patient from host arrays (uploads, kernels, downloads, the .npy / pickle writes), a host clock around a call
  that ends in a synchronise; the reader returns arrays already in memory, so file reading is excluded;
- `read_npy_s`: reading the same 13 volumes back from .npy files, for scale: reading .nrrd / .nii.gz with SimpleITK is not measured here
  and is likely to cost more than the preprocessing;
- `scipy_ct_s`, `scipy_rater_s`: oracle/preprocess_oracle.py (scipy.ndimage, fp64) for one CT and one rater on one host core;
  `scipy_patient_s` = scipy_ct_s + 12 scipy_rater_s, derived from those two, not timed as a whole.

    python tools/preprocess_bench.py [--reps 10] [--no-scipy]"""
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
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import preprocess_oracle as PO  # noqa: E402
from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import preprocessing as P  # noqa: E402
from medicaldetectiontoolkit_b200.configs import make_cf  # noqa: E402

KINDS = {"up_z": ((250, 512, 512), (0.65, 0.65, 2.5)), "down": ((400, 512, 512), (0.55, 0.55, 1.0))}
PIDS = {"up_z": "LIDC-IDRI-0901", "down": "LIDC-IDRI-0902"}
TARGET = (0.7, 0.7, 1.25)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def make_patient(shape, seed):
    rs = np.random.RandomState(seed)
    ct = (rs.normal(-500, 400, shape)).astype(np.int16)
    rois = []
    for r in range(3):
        c = [rs.randint(s // 4, 3 * s // 4) for s in shape]
        raters = []
        for _ in range(4):
            z, y, x = np.ogrid[:shape[0], :shape[1], :shape[2]]
            rad = rs.uniform(4, 9, 3)
            cc = [ci + rs.randint(-2, 3) for ci in c]
            raters.append((((z - cc[0]) / rad[0]) ** 2 + ((y - cc[1]) / rad[1]) ** 2 + ((x - cc[2]) / rad[2]) ** 2 <= 1).astype(np.uint8))
        rois.append(raters)
    return ct, rois


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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-scipy", action="store_true")
    a = ap.parse_args()
    emit(card=card(), torch=torch.__version__)
    ops = P.CudaOps("cuda:0")
    for kind, (shape, spacing) in KINDS.items():
        ct, rois = make_patient(shape, 1)
        out_shape = P.target_shape(shape, spacing, TARGET)
        ct_dev = ops.upload(ct)
        raters_dev = [ops.upload(r) for r in rois[0]]
        img = torch.empty(out_shape, dtype=torch.float32, device="cuda:0")

        def ct_step():
            ops.resample(ct_dev, out_shape, out=img)
            ops.normalize(img)
        state = ops.begin(ct, out_shape)
        state["acc"], state["rater"] = torch.empty_like(img), torch.empty_like(img)

        def roi_step():
            lib = L.load()
            for k, r in enumerate(raters_dev):
                ops.resample(r, out_shape, out=state["rater"])
                L.check(lib.mdt_pp_vote_add(L.ptr(state["acc"]), L.ptr(state["rater"]), img.numel(), int(k == 0), L.stream_ptr()))
            L.check(lib.mdt_pp_vote_label(L.ptr(state["acc"]), img.numel(), 4, 0, L.ptr(state["labels"]), L.ptr(state["kept"]), L.stream_ptr()))
        ct_ms = device_ms(ct_step, a.reps)
        roi_ms = device_ms(roi_step, a.reps)
        del state

        with tempfile.TemporaryDirectory() as tmp:
            pid = PIDS[kind]
            raw = os.path.join(tmp, "data_nrrd")
            pdir = os.path.join(raw, pid)
            os.makedirs(pdir)
            files = {"%s_ct_scan.nrrd" % pid: ct}
            rows = ["PatientID;NoduleID;Malignancy"]
            for r, raters in enumerate(rois):
                for k, arr in enumerate(raters):
                    nid = 10 * (r + 1) + k
                    files["%s_nod_%04d_%d.nii.gz" % (pid, nid, r + 1)] = arr
                    rows.append("%s;%d;%d" % (pid, nid, 1 + (nid % 5)))
            for name in files:
                open(os.path.join(pdir, name), "wb").close()
            with open(os.path.join(tmp, "characteristics.csv"), "w") as f:
                f.write("\n".join(rows) + "\n")
            cf = make_cf(exp="lidc_exp")
            cf.root_dir, cf.raw_data_dir, cf.pp_dir = tmp, raw, os.path.join(tmp, "pp")
            os.makedirs(cf.pp_dir)

            def reader(path):
                return files[os.path.basename(path)], spacing
            P.pp_patient((0, pdir), cf, read_image=reader, ops=ops)        # warm-up
            times = []
            for _ in range(3):
                torch.cuda.synchronize()
                t = time.perf_counter()
                P.pp_patient((0, pdir), cf, read_image=reader, ops=ops)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t)
            npy = os.path.join(tmp, "npy")
            os.makedirs(npy)
            for name, arr in files.items():
                np.save(os.path.join(npy, name + ".npy"), arr)
            t = time.perf_counter()
            for name in files:
                np.load(os.path.join(npy, name + ".npy"))
            read_s = time.perf_counter() - t          # the page cache may hold these files: a lower bound on reading
        rec = dict(kind=kind, shape=list(shape), out_shape=out_shape, ct_ms=round(ct_ms, 3), roi_ms=round(roi_ms, 3),
                   patient_s=round(float(np.median(times)), 4), read_npy_s=round(read_s, 4))
        if not a.no_scipy:
            t = time.perf_counter()
            PO.normalize(PO.resample_array(ct, spacing, TARGET))
            rec["scipy_ct_s"] = round(time.perf_counter() - t, 2)
            t = time.perf_counter()
            PO.resample_array(rois[0][0], spacing, TARGET)
            rec["scipy_rater_s"] = round(time.perf_counter() - t, 2)
            rec["scipy_patient_s"] = round(rec["scipy_ct_s"] + 12 * rec["scipy_rater_s"], 2)
        emit(**rec)


if __name__ == "__main__":
    main()
