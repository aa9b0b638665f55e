#!/usr/bin/env python
"""Times the patient bootstrap of the evaluator on a synthetic lidc 3D test set: 200 patients, 2 classes, 3 match IoUs, 30 detections per
class and patient (0-3 GT boxes each), matched by evaluate_predictions.  For n_resamples = 1000 and 10 000 (plus the point estimate):
  - the device time of mdt_eval_bootstrap_roi and mdt_eval_bootstrap_patient alone (CUDA events around warmed-up calls on resident
    buffers, the mean of --reps calls);
  - the whole Evaluator.bootstrap call (host clock, ending in a device synchronise: draws, uploads, kernels, copy back, host reductions);
  - the materialising numpy oracle (tests/_bootstrap_oracle.py) per resample on one host core, timed on --oracle-resamples resamples.
Prints one JSON line per n_resamples, with the card, its power limit and max SM clock read in the same run.
Usage: python tools/eval_bootstrap_bench.py [--reps N] [--oracle-resamples N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bootstrap_oracle as B  # noqa: E402
from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import evaluator as E  # noqa: E402
from medicaldetectiontoolkit_b200.configs import make_cf  # noqa: E402


class _Log:
    def info(self, *a, **k):
        pass


def _box(rs, extent=128.0):
    c = rs.uniform(30, extent - 30, size=3)
    s = rs.uniform(4, 30, size=3)
    a, b = c - s / 2, c + s / 2
    return np.array([a[0], a[1], b[0], b[1], a[2], b[2]])


def test_set(n_pat=200, n_det=30):
    rs = np.random.RandomState(0)
    res = []
    for p in range(n_pat):
        boxes = []
        for cl in (1, 2):
            gts = [_box(rs) for _ in range(rs.randint(0, 4))]
            boxes += [{'box_coords': g, 'box_type': 'gt', 'box_label': cl} for g in gts]
            for _ in range(n_det):
                d = gts[rs.randint(len(gts))] + rs.normal(0, 3, size=6) if gts and rs.rand() < 0.3 else _box(rs)
                boxes.append({'box_coords': d, 'box_type': 'det', 'box_score': float(rs.rand()), 'box_pred_class_id': cl})
        res.append([[boxes], 'p%03d' % p])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--oracle-resamples', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bootstrap_bench measures the GPU kernels: no CUDA device")
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})        # one host core, for the oracle and the host part alike
    torch.set_num_threads(1)
    cf = make_cf('retina_unet', 3)
    cf.ap_match_ious = [0.1, 0.25, 0.5]
    ev = E.Evaluator(cf, _Log(), 'test')
    ev.evaluate_predictions(test_set())
    c = ev.columns
    roi, pat, pat_idx, n_pat = E._bootstrap_jobs(c, list(cf.class_dict.keys()), list(cf.report_score_level))
    lib = L.load()
    dev = torch.device('cuda', 0)
    idx = np.concatenate(roi.rows)
    n_roi, n_all = int(idx.size), int(c['pred_score'].size)
    n_members = sum(m.size for m in pat.members)
    seg_off = np.concatenate([[0], np.cumsum([m.size for m in pat.members])]).astype(np.int32)
    rates = np.array(E.FROC_RATES, dtype=np.float64)

    def d(a, dt):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
    r_in = [d(c['pred_score'][idx], np.float64), d(np.concatenate(roi.segs), np.int32), d(roi.codes[idx], np.int32), d(pat_idx[idx], np.int32),
            d(E.RECALL_POINTS, np.float64), d(rates * n_pat, np.float64)]
    p_in = [d(c['pred_score'], np.float64), d(c['class_label'], np.int32), d(pat.row_slot, np.int32), d(pat_idx, np.int32), d(seg_off, np.int32),
            d(np.concatenate(pat.members), np.int32)]
    for n_res in (1000, 10000):
        mult = np.concatenate([np.ones((1, n_pat), np.int32), E.draw_multiplicities(n_pat, n_res, 0)])
        nb = mult.shape[0]
        m = d(mult, np.int32)
        n_r = E.RECALL_POINTS.size
        q = torch.empty(nb * roi.n_seg * n_r, dtype=torch.float64, device=dev)
        cnt = torch.empty(nb * roi.n_seg * 2, dtype=torch.int32, device=dev)
        fr = torch.empty(nb * roi.n_seg * rates.size, dtype=torch.int32, device=dev)
        thr = torch.empty(nb * n_members, dtype=torch.float64, device=dev)
        tps = torch.empty(nb * n_members, dtype=torch.int32, device=dev)
        fps = torch.empty(nb * n_members, dtype=torch.int32, device=dev)
        n_thr = torch.empty(nb * len(pat.members), dtype=torch.int32, device=dev)
        rws = torch.empty(lib.mdt_eval_bootstrap_roi_workspace_bytes(n_roi, roi.n_seg, n_pat), dtype=torch.uint8, device=dev)
        pws = torch.empty(lib.mdt_eval_bootstrap_patient_workspace_bytes(pat.n_slots, n_members, len(pat.members)), dtype=torch.uint8, device=dev)
        stream = L.stream_ptr()

        def run_roi():
            L.check(lib.mdt_eval_bootstrap_roi(*[L.ptr(t) for t in r_in[:4]], n_roi, roi.n_seg, n_pat, L.ptr(m), nb, float(cf.min_det_thresh),
                                               L.ptr(r_in[4]), n_r, L.ptr(r_in[5]), rates.size, L.ptr(q), L.ptr(cnt), L.ptr(fr), L.ptr(rws),
                                               rws.numel(), stream))

        def run_pat():
            L.check(lib.mdt_eval_bootstrap_patient(*[L.ptr(t) for t in p_in[:4]], n_all, pat.n_slots, L.ptr(p_in[4]), L.ptr(p_in[5]), n_members,
                                                   len(pat.members), n_pat, L.ptr(m), nb, L.ptr(thr), L.ptr(tps), L.ptr(fps), L.ptr(n_thr),
                                                   L.ptr(pws), pws.numel(), stream))
        times = {}
        for name, fn in (('roi', run_roi), ('patient', run_pat)):
            fn()
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.reps):
                fn()
            end.record()
            torch.cuda.synchronize()
            times[name] = start.elapsed_time(end) / 1e3 / args.reps
        ev.bootstrap(n_resamples=n_res)                                    # warm-up of the whole call
        t0 = time.perf_counter()
        stats = ev.bootstrap(n_resamples=n_res)
        torch.cuda.synchronize()
        t_call = time.perf_counter() - t0
        k = args.oracle_resamples
        t0 = time.perf_counter()
        B.run_bootstrap_kernels(roi, pat, pat_idx, n_pat, mult[1:1 + k], cf.min_det_thresh, rates * n_pat)
        t_oracle = (time.perf_counter() - t0) / k
        avg = stats[-1]['ap']
        print(json.dumps({'n_resamples': n_res, 'card': card, 'patients': int(n_pat), 'rows': n_all, 'roi_rows': n_roi,
                          'roi_segments': roi.n_seg, 'patient_members': int(n_members),
                          'roi_kernel_s': round(times['roi'], 5), 'patient_kernel_s': round(times['patient'], 5),
                          'bootstrap_call_s': round(t_call, 3), 'oracle_1core_s_per_resample': round(t_oracle, 4),
                          'oracle_resamples_timed': k, 'average_foreground_roi_ap': [avg['value'], list(avg['ci']), avg['n_valid']]}), flush=True)


if __name__ == '__main__':
    main()
