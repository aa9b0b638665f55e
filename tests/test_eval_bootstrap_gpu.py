"""The patient bootstrap and FROC on the GPU (csrc/evaluate.cu: mdt_eval_bootstrap_roi, mdt_eval_bootstrap_patient) against the materialising
numpy oracle (tests/_bootstrap_oracle.py), bit for bit: every golden case of tests/golden/evaluator.pkl.gz, adversarial ties, and a
workload-scale test set.  With every multiplicity 1 the point estimates equal return_metrics'.  Each entry point through poisoned exact-size
buffers, their error statuses, determinism, chunking, and score_bootstrap's file."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bootstrap_oracle as B  # noqa: E402
import make_eval_golden as G  # noqa: E402
from _guarded import _run_guarded  # noqa: E402
from test_eval_bootstrap_cpu import _check_score_bootstrap_text, _same  # noqa: E402

from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import evaluator as E  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RATES = np.array(E.FROC_RATES, dtype=np.float64)


def _d(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(DEV)


def _evaluator(name):
    ev, _ = G.run_case(E, name)
    ev.cf.per_patient_ap = False
    ev.cf.scan_det_thresh = False
    return ev


def _jobs(ev):
    return E._bootstrap_jobs(ev.columns, list(ev.cf.class_dict.keys()), list(ev.cf.report_score_level))


def _check_res(got, want, pat, rows=None):
    """kernel outputs (optionally only resamples `rows`) equal the oracle's; patient curves compared where they are written"""
    sel = slice(None) if rows is None else rows
    for k in ('q', 'counts', 'froc'):
        assert (k in got) == (k in want)
        if k in got:
            assert np.array_equal(got[k][sel], want[k]), k
    if pat.members:
        off = np.concatenate([[0], np.cumsum([m.size for m in pat.members])])
        n_thr = got['n_thr'][sel]
        assert np.array_equal(n_thr, want['n_thr'])
        for b in range(n_thr.shape[0]):
            for k in range(len(pat.members)):
                s = slice(off[k], off[k] + n_thr[b, k])
                for name in ('thr', 'tps', 'fps'):
                    assert np.array_equal(got[name][sel][b, s], want[name][b, s]), (name, b, k)


# -------------------------------------------------------------------------------------------------------------- identity
@pytest.mark.parametrize("name", G.CASES)
def test_point_estimates_equal_return_metrics(name):
    ev = _evaluator(name)
    want, _ = ev.return_metrics(None if ev.mode == 'test' else G.new_monitor_metrics(ev.cf))
    got = ev.bootstrap(n_resamples=0)
    assert [g['name'] for g in got] == [w['name'] for w in want]
    for g, w in zip(got, want):
        assert _same([g['ap']['value']], [w['ap']]), g['name']
        if 'patient' in g['name']:
            assert _same([g['auc']['value']], [w['auc']]), g['name']


# ---------------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize("name", G.CASES)
def test_golden_cases_64_resamples_equal_the_materialising_oracle(name):
    ev = _evaluator(name)
    roi, pat, pat_idx, n_pat = _jobs(ev)
    mult = np.concatenate([np.ones((1, n_pat), np.int32), E.draw_multiplicities(n_pat, 64, 0)])
    args = (roi, pat, pat_idx, n_pat, mult, ev.cf.min_det_thresh, RATES * n_pat)
    _check_res(E._run_bootstrap_kernels(*args), B.run_bootstrap_kernels(*args), pat)
    got = ev.bootstrap(n_resamples=64)
    got_v = ev.bootstrap_values
    undo = B.patch(E)
    try:
        want = ev.bootstrap(n_resamples=64)
    finally:
        undo()
    assert repr(got) == repr(want)
    assert repr(got_v) == repr(ev.bootstrap_values)


def _tie_rows():
    """adversarial ties: TP and FP rows of one patient at one score, equal scores across patients and across cub sort tiles (20 000
    rows on a 0.05 grid), rows exactly at the threshold, NaN scores, FNs and patient_tn rows"""
    rs = np.random.RandomState(7)
    n, n_pat, n_seg = 20000, 50, 3
    score = np.round(rs.uniform(0, 1, n) / 0.05) * 0.05
    score[rs.rand(n) < 0.02] = np.nan
    score[rs.rand(n) < 0.02] = 0.1
    kind = rs.choice([0, 1, 2, 3], n, p=[0.3, 0.5, 0.15, 0.05]).astype(np.int32)
    score[kind >= 2] = 0.0
    seg = np.where(kind == 3, -1, rs.randint(0, n_seg, n)).astype(np.int32)
    patient = rs.randint(0, n_pat, n).astype(np.int32)
    same = np.nonzero(patient == 3)[0][:6]               # patient 3: TP and FP at one score
    kind[same], score[same], seg[same] = [0, 1, 0, 1, 1, 0], 0.55, 1
    mult = [np.ones(n_pat, np.int32), np.zeros(n_pat, np.int32), np.zeros(n_pat, np.int32)]
    mult[2][3] = n_pat                                    # one patient drawn P times
    mult += [B.draw(5, b, n_pat) for b in range(5)]
    z = B.draw(6, 0, n_pat)
    z[::3] = 0                                            # zero-weight patients (and sums != P)
    mult.append(z)
    return score, seg, kind, patient, n_pat, n_seg, np.array(mult, dtype=np.int32)


def _roi_call(score, seg, kind, patient, n_pat, n_seg, mult, lim, th=0.1):
    lib = L.load()
    n, nb, R = score.size, mult.shape[0], E.RECALL_POINTS
    ws_b = lib.mdt_eval_bootstrap_roi_workspace_bytes(n, n_seg, n_pat)
    assert ws_b > 0
    d = [_d(score, np.float64), _d(seg, np.int32), _d(kind, np.int32), _d(patient, np.int32), _d(mult, np.int32), _d(R, np.float64),
         _d(lim, np.float64)]

    def call(outs, ws):
        return lib.mdt_eval_bootstrap_roi(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), n, n_seg, n_pat, L.ptr(d[4]), nb, th,
                                          L.ptr(d[5]), R.size, L.ptr(d[6]), lim.size, outs[0], outs[1], outs[2], ws, ws_b, None)
    return call, [8 * nb * n_seg * R.size, 4 * nb * n_seg * 2, 4 * nb * n_seg * lim.size], ws_b


def test_roi_entry_adversarial_ties_guarded():
    score, seg, kind, patient, n_pat, n_seg, mult = _tie_rows()
    lim = RATES * n_pat
    call, sizes, ws_b = _roi_call(score, seg, kind, patient, n_pat, n_seg, mult, lim)
    got = _run_guarded(call, sizes, ws_b)
    q, counts, tp = B.bootstrap_roi(score, seg, kind, patient, n_seg, mult, 0.1, E.RECALL_POINTS, lim)
    assert np.array_equal(got[0].view(torch.float64).cpu().numpy().reshape(q.shape), q)
    assert np.array_equal(got[1].view(torch.int32).cpu().numpy().reshape(counts.shape), counts)
    assert np.array_equal(got[2].view(torch.int32).cpu().numpy().reshape(tp.shape), tp)
    assert counts[1].sum() == 0 and not q[1].any()        # every weight 0


def _pat_call(score, label, slot, patient, n_slots, members, n_pat, mult):
    lib = L.load()
    off = np.concatenate([[0], np.cumsum([m.size for m in members])]).astype(np.int32)
    n, n_mem, nb, n_seg = score.size, int(off[-1]), mult.shape[0], len(members)
    ws_b = lib.mdt_eval_bootstrap_patient_workspace_bytes(n_slots, n_mem, n_seg)
    assert ws_b > 0
    d = [_d(score, np.float64), _d(label, np.int32), _d(slot, np.int32), _d(patient, np.int32), _d(off, np.int32),
         _d(np.concatenate(members), np.int32), _d(mult, np.int32)]

    def call(outs, ws):
        return lib.mdt_eval_bootstrap_patient(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), n, n_slots, L.ptr(d[4]), L.ptr(d[5]), n_mem,
                                              n_seg, n_pat, L.ptr(d[6]), nb, outs[0], outs[1], outs[2], outs[3], ws, ws_b, None)
    return call, [8 * nb * n_mem, 4 * nb * n_mem, 4 * nb * n_mem, 4 * nb * n_seg], ws_b, off


def test_patient_entry_adversarial_ties_guarded():
    rs = np.random.RandomState(9)
    n_pat, n_slots, n = 300, 600, 4000
    slot_pat = np.concatenate([np.arange(300), np.arange(300)]).astype(np.int32)   # slot s: class s // 300 of patient s % 300
    slot = rs.randint(-1, n_slots, n).astype(np.int32)
    slot[:n_slots] = np.arange(n_slots)
    slot[5] = 7                                                                    # slot 7 gets two rows
    patient = np.where(slot >= 0, slot_pat[np.maximum(slot, 0)], rs.randint(0, n_pat, n)).astype(np.int32)
    score = np.round(rs.uniform(0, 1, n), 1)                                       # ties within and across patients
    score[rs.rand(n) < 0.3] = 0.0
    label = (rs.rand(n) < 0.25).astype(np.int32)
    members = [np.arange(0, 300, dtype=np.int32), np.arange(300, 600, dtype=np.int32), np.array([3, 9, 303, 450], dtype=np.int32),
               np.arange(0, 600, 2, dtype=np.int32)]
    mult = [np.ones(n_pat, np.int32), np.zeros(n_pat, np.int32), np.zeros(n_pat, np.int32)]
    mult[2][9] = n_pat
    mult += [B.draw(2, b, n_pat) for b in range(4)]
    mult = np.array(mult, dtype=np.int32)
    call, sizes, ws_b, off = _pat_call(score, label, slot, patient, n_slots, members, n_pat, mult)
    got = _run_guarded(call, sizes, ws_b, out_fills=(0xFF,))
    want = B.bootstrap_patient(score, label, slot, patient, n_slots, members, mult)
    n_mem = int(off[-1])
    thr = got[0].view(torch.float64).cpu().numpy().reshape(-1, n_mem)
    tps = got[1].view(torch.int32).cpu().numpy().reshape(-1, n_mem)
    fps = got[2].view(torch.int32).cpu().numpy().reshape(-1, n_mem)
    n_thr = got[3].view(torch.int32).cpu().numpy().reshape(-1, len(members))
    for b, wb in enumerate(want):
        for k, (u, tp, fp) in enumerate(wb):
            assert n_thr[b, k] == u.size, (b, k)
            s = slice(off[k], off[k] + u.size)
            assert np.array_equal(thr[b, s], u) and np.array_equal(tps[b, s], tp) and np.array_equal(fps[b, s], fp), (b, k)
    assert (n_thr[1] == 0).all()


def _scale_results(rs, n_pat=200, n_det=80):
    res = []
    for p in range(n_pat):
        boxes = []
        for cl in (1, 2):
            gts = [G._box(rs, 3, 128.0) for _ in range(rs.randint(0, 4))]
            boxes += [{'box_coords': g, 'box_type': 'gt', 'box_label': cl} for g in gts]
            for _ in range(n_det):
                d = gts[rs.randint(len(gts))] + rs.normal(0, 2, 6) if gts and rs.rand() < 0.3 else G._box(rs, 3, 128.0)
                boxes.append({'box_coords': d, 'box_type': 'det', 'box_score': float(np.round(rs.rand(), 3)), 'box_pred_class_id': cl})
        res.append([[boxes], 'p%03d' % p])
    return res


def test_workload_scale_equals_the_oracle_on_sampled_resamples():
    cf = G.base_cf(ap_match_ious=[0.1, 0.25, 0.5])
    ev = E.Evaluator(cf, G.Logger(), 'test')
    ev.evaluate_predictions(_scale_results(np.random.RandomState(0)))
    assert ev.columns['pred_score'].size > 90000
    roi, pat, pat_idx, n_pat = _jobs(ev)
    mult = np.concatenate([np.ones((1, n_pat), np.int32), E.draw_multiplicities(n_pat, 1000, 0)])
    args = (roi, pat, pat_idx, n_pat)
    got = E._run_bootstrap_kernels(*args, mult, cf.min_det_thresh, RATES * n_pat)
    sample = np.array([0, 1, 2, 137, 500, 999, 1000])
    want = B.run_bootstrap_kernels(*args, mult[sample], cf.min_det_thresh, RATES * n_pat)
    _check_res(got, want, pat, rows=sample)


# ---------------------------------------------------------------------------------------------- guarded golden, errors, runs
def test_golden_rows_through_guarded_buffers():
    ev = _evaluator('train_3d')
    roi, pat, pat_idx, n_pat = _jobs(ev)
    mult = E.draw_multiplicities(n_pat, 5, 3)
    idx = np.concatenate(roi.rows)
    c = ev.columns
    lim = RATES * n_pat
    call, sizes, ws_b = _roi_call(c['pred_score'][idx], np.concatenate(roi.segs), roi.codes[idx], pat_idx[idx], n_pat, roi.n_seg, mult, lim)
    got = _run_guarded(call, sizes, ws_b)
    q, counts, tp = B.bootstrap_roi(c['pred_score'][idx], np.concatenate(roi.segs), roi.codes[idx], pat_idx[idx], roi.n_seg, mult, 0.1,
                                    E.RECALL_POINTS, lim)
    assert np.array_equal(got[0].view(torch.float64).cpu().numpy().reshape(q.shape), q)
    assert np.array_equal(got[1].view(torch.int32).cpu().numpy().reshape(counts.shape), counts)
    assert np.array_equal(got[2].view(torch.int32).cpu().numpy().reshape(tp.shape), tp)
    call, sizes, ws_b, off = _pat_call(c['pred_score'], c['class_label'], pat.row_slot, pat_idx, pat.n_slots, pat.members, n_pat, mult)
    _run_guarded(call, sizes, ws_b, out_fills=(0xFF,))


def test_entry_points_return_error_statuses():
    lib = L.load()
    buf = torch.zeros(1 << 20, dtype=torch.int32, device=DEV)
    p = L.ptr(buf)
    big = 1 << 20
    ws_b = lib.mdt_eval_bootstrap_roi_workspace_bytes(4, 1, 2)

    def roi(n=4, n_seg=1, P=2, nb=1, n_r=101, n_rates=7, ws=ws_b):
        return lib.mdt_eval_bootstrap_roi(p, p, p, p, n, n_seg, P, p, nb, 0.1, p, n_r, p, n_rates, p, p, p, p, ws, None)
    assert roi(n_r=129) == -1
    assert roi(n_rates=129) == -1 and roi(n_rates=0) == -1
    assert roi(n=-1) == -1 and roi(nb=-1) == -1 and roi(P=0) == -1 and roi(n_seg=0) == -1
    assert roi(n=big, P=1 << 11) == -1                      # n_patients * n_rows = 2^31
    assert roi(ws=ws_b - 1) == -2
    assert roi() == 0                                       # zeros: patient 0 of 2, multiplicity 0
    pats = _d(np.array([0, 1, 2, 0]), np.int32)             # patient index 2 of P = 2
    assert lib.mdt_eval_bootstrap_roi(p, p, p, L.ptr(pats), 4, 1, 2, p, 1, 0.1, p, 101, p, 7, p, p, p, p, ws_b, None) == -1
    negm = _d(np.array([1, -1]), np.int32)
    assert lib.mdt_eval_bootstrap_roi(p, p, p, p, 4, 1, 2, L.ptr(negm), 1, 0.1, p, 101, p, 7, p, p, p, p, ws_b, None) == -1
    pws = lib.mdt_eval_bootstrap_patient_workspace_bytes(4, 4, 1)

    def patient(n=4, n_slots=4, n_mem=4, n_seg=1, P=2, nb=1, ws=pws, pt=p, m=p):
        return lib.mdt_eval_bootstrap_patient(p, p, p, pt, n, n_slots, p, p, n_mem, n_seg, P, m, nb, p, p, p, p, p, ws, None)
    assert patient(n=-1) == -1 and patient(n_slots=0) == -1 and patient(nb=-1) == -1 and patient(P=-1) == -1
    assert patient(n=big, P=1 << 11) == -1
    assert patient(ws=pws - 1) == -2
    assert patient() == 0
    assert patient(pt=L.ptr(pats)) == -1 and patient(m=L.ptr(negm)) == -1
    torch.cuda.synchronize()


def test_python_arguments_raise():
    ev = _evaluator('edges')
    for kw in (dict(n_resamples=-1), dict(alpha=0), dict(alpha=1.5), dict(fps_per_scan=(0.5, -1)), dict(fps_per_scan=(np.nan,))):
        with pytest.raises(ValueError):
            ev.bootstrap(**kw)


def test_two_runs_and_smaller_chunks_are_bit_identical(monkeypatch):
    ev = _evaluator('test_plain')
    a = ev.bootstrap(n_resamples=200, seed=3)
    va = repr(ev.bootstrap_values)
    b = ev.bootstrap(n_resamples=200, seed=3)
    assert repr(a) == repr(b) and va == repr(ev.bootstrap_values)
    monkeypatch.setattr(E, 'BOOTSTRAP_CHUNK_BYTES', 50000)
    c = ev.bootstrap(n_resamples=200, seed=3)
    assert repr(a) == repr(c) and va == repr(ev.bootstrap_values)


def test_score_bootstrap_file(tmp_path):
    pytest.importorskip('pandas')
    _check_score_bootstrap_text(tmp_path)
