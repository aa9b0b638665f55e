"""numpy oracle of the patient bootstrap and the FROC (medicaldetectiontoolkit_b200/csrc/evaluate.cu, mdt_eval_bootstrap_roi /
mdt_eval_bootstrap_patient).  The bootstrap here materialises every resample: each row of patient p repeated m[p] times in place (np.repeat,
copies next to each other), copy j of p a patient of its own, and then runs oracle/eval_oracle.py's roi_ap / patient_counts and froc()
below on the repeated rows.  Test infrastructure only: nothing in the package imports it."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import eval_oracle as O  # noqa: E402


def draw(seed, b, n_pat):
    """the multiplicities of resample b: np.bincount of RandomState([seed, b]).randint(0, P, P)"""
    return np.bincount(np.random.RandomState([seed, b]).randint(0, n_pat, size=n_pat), minlength=n_pat).astype(np.int32)


def froc(score, seg, kind, n_seg, threshold, fp_limits):
    """step FROC per segment: (sens [n_seg, n_rates], tp [n_seg, n_rates], G [n_seg]).  G = det_tp + det_fn rows; the operating points
    are the origin and, per distinct score v of the det_tp / det_fp rows with a non-NaN score > threshold, (TP(v), FP(v)) = the TP / FP
    detections with score >= v; tp[f] = max{TP(v) : FP(v) <= fp_limits[f]}; sens = tp / G, NaN when G = 0"""
    score, seg, kind = np.asarray(score, dtype=np.float64), np.asarray(seg), np.asarray(kind)
    lim = np.asarray(fp_limits, dtype=np.float64)
    tp = np.zeros((n_seg, lim.size), dtype=np.int64)
    G = np.zeros(n_seg, dtype=np.int64)
    for s in range(n_seg):
        G[s] = np.count_nonzero((seg == s) & ((kind == 0) | (kind == 2)))
        det = (seg == s) & ((kind == 0) | (kind == 1)) & ~np.isnan(score)
        det &= np.where(det, score, -np.inf) > threshold
        sc, is_tp = score[det], kind[det] == 0
        v = np.unique(sc)
        s_tp, s_fp = np.sort(sc[is_tp]), np.sort(sc[~is_tp])
        TP = np.concatenate([[0], s_tp.size - np.searchsorted(s_tp, v, 'left')])      # the origin, then every distinct score
        FP = np.concatenate([[0], s_fp.size - np.searchsorted(s_fp, v, 'left')])
        tp[s] = [TP[FP <= x].max() for x in lim]
    with np.errstate(invalid='ignore', divide='ignore'):
        sens = np.where(G[:, None] > 0, tp / np.maximum(G, 1)[:, None].astype(np.float64), np.nan)
    return sens, tp, G


def materialise(n_rows, row_patient, mult):
    """(idx, copy): the row indices of the materialised resample (np.repeat in place) and each repeated row's copy number j"""
    w = np.asarray(mult)[np.asarray(row_patient)]
    idx = np.repeat(np.arange(n_rows), w)
    start = np.concatenate([[0], np.cumsum(w)[:-1]]) if n_rows else np.zeros(0, dtype=np.int64)
    copy = np.arange(idx.size) - np.repeat(start, w)
    return idx, copy


def bootstrap_roi(score, seg, kind, patient, n_seg, mult, threshold, recall_points, fp_limits):
    """mdt_eval_bootstrap_roi on the materialised resamples: q [n_boot, n_seg, n_r], counts [n_boot, n_seg, 2], froc_tp [n_boot, n_seg, n_rates]"""
    mult = np.atleast_2d(mult)
    qs, cs, fs = [], [], []
    for m in mult:
        idx, _ = materialise(score.size, patient, m)
        q, counts = O.roi_ap(score[idx], seg[idx], kind[idx], n_seg, [threshold], recall_points)
        _, tp, _ = froc(score[idx], seg[idx], kind[idx], n_seg, threshold, fp_limits)
        qs.append(q[:, 0])
        cs.append(counts)
        fs.append(tp)
    return np.array(qs), np.array(cs, dtype=np.int32), np.array(fs, dtype=np.int32)


def bootstrap_patient(score, label, slot, patient, n_slots, members, mult):
    """mdt_eval_bootstrap_patient on the materialised resamples: per resample the patient_counts list [(thr, tps, fps) per segment].
    Copy j of slot s is the new slot s * (P + 1) + j (P >= any multiplicity), and a member slot becomes its m copies."""
    mult = np.atleast_2d(mult)
    out = []
    slot = np.asarray(slot)
    slot_pat = np.full(n_slots, -1)
    ok = slot >= 0
    slot_pat[slot[ok]] = np.asarray(patient)[ok]
    n_pat = mult.shape[1]
    for m in mult:
        idx, copy = materialise(score.size, patient, m)
        s = slot[idx]
        s_new = np.where(s >= 0, s * (n_pat + 1) + copy, -1)
        mem = []
        for mm in members:
            mm = np.asarray(mm)
            k = np.where(slot_pat[mm] >= 0, m[np.maximum(slot_pat[mm], 0)], 0)
            mem.append(np.repeat(mm * (n_pat + 1), k) + np.concatenate([np.arange(x) for x in k]).astype(np.int64) if k.sum() else
                       np.zeros(0, dtype=np.int64))
        out.append(O.patient_counts(score[idx], label[idx], s_new, n_slots * (n_pat + 1), mem))
    return out


def run_bootstrap_kernels(roi, pat, pat_idx, n_pat, mult, threshold, fp_limits):
    """the oracle counterpart of evaluator._run_bootstrap_kernels (same inputs, same result dict), on materialised resamples"""
    from medicaldetectiontoolkit_b200.evaluator import RECALL_POINTS
    mult = np.atleast_2d(mult)
    res = {}
    if roi.n_seg:
        idx = np.concatenate(roi.rows)
        res['q'], res['counts'], res['froc'] = bootstrap_roi(roi.c['pred_score'][idx], np.concatenate(roi.segs), roi.codes[idx], pat_idx[idx],
                                                             roi.n_seg, mult, threshold, RECALL_POINTS, fp_limits)
    if pat.members:
        n_members = sum(m.size for m in pat.members)
        off = np.concatenate([[0], np.cumsum([m.size for m in pat.members])])
        res['thr'] = np.zeros((mult.shape[0], n_members))
        res['tps'] = np.zeros((mult.shape[0], n_members), dtype=np.int32)
        res['fps'] = np.zeros((mult.shape[0], n_members), dtype=np.int32)
        res['n_thr'] = np.zeros((mult.shape[0], len(pat.members)), dtype=np.int32)
        curves = bootstrap_patient(pat.c['pred_score'], pat.c['class_label'], pat.row_slot, pat_idx, max(pat.n_slots, 1), pat.members, mult)
        for b, cb in enumerate(curves):
            for k, (u, tp, fp) in enumerate(cb):
                sl = slice(off[k], off[k] + u.size)
                res['thr'][b, sl], res['tps'][b, sl], res['fps'][b, sl] = u, tp, fp
                res['n_thr'][b, k] = u.size
    return res


def patch(evaluator_module):
    """run medicaldetectiontoolkit_b200.evaluator's bootstrap on this oracle and its other metrics on oracle/eval_oracle.py (returns an undo)"""
    undo_eval = O.patch(evaluator_module)
    saved = evaluator_module._run_bootstrap_kernels
    evaluator_module._run_bootstrap_kernels = run_bootstrap_kernels

    def undo():
        evaluator_module._run_bootstrap_kernels = saved
        undo_eval()
    return undo
