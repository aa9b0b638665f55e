"""numpy-only restatement of the evaluation kernels (medicaldetectiontoolkit_b200/csrc/evaluate.cu) in their formulation: the rows of one
(IoU, class, patient) slot in the kernels' emission order, stable score order (ties in row order), integer counts and then divisions.
No pandas and no scikit-learn.  Each function takes and returns what the corresponding host call of medicaldetectiontoolkit_b200/evaluator.py
(match_rows, _run_metric_kernels) takes and returns, so the Evaluator runs on it unchanged: the CPU model of the kernels, pinned to the
reference's goldens in tests/test_evaluator_cpu.py, and the host baseline of tools/eval_bench.py."""
import numpy as np


def _iou_rows(cand, gt, dim):
    """compute_overlaps(cand, gt) [n_cand, n_gt]: per GT column, the reference's operation order"""
    def vol(b):
        v = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
        return v * (b[:, 5] - b[:, 4]) if dim == 3 else v
    vc, vg = vol(cand), vol(gt)
    out = np.zeros((cand.shape[0], gt.shape[0]))
    with np.errstate(divide='ignore', invalid='ignore'):
        for j in range(gt.shape[0]):
            g = gt[j]
            inter = np.maximum(np.minimum(g[3], cand[:, 3]) - np.maximum(g[1], cand[:, 1]), 0) * \
                np.maximum(np.minimum(g[2], cand[:, 2]) - np.maximum(g[0], cand[:, 0]), 0)
            if dim == 3:
                inter = inter * np.maximum(np.minimum(g[5], cand[:, 5]) - np.maximum(g[4], cand[:, 4]), 0)
            out[:, j] = inter / (vg[j] + vc - inter)
    return out


def _beats(si, sb):
    return (not np.isnan(sb)) if np.isnan(si) else si > sb


def match_rows(flat, n_classes, ious):
    """mdt_eval_match: (row_score, row_meta [n, 4] = type, class index, patient index, IoU index)"""
    dim, cand, score, cand_off, gt, gt_off, elem_off = flat
    rs, rm = [], []
    for iu, t in enumerate(ious):
        for cl in range(n_classes):
            for p in range(elem_off.size - 1):
                start = len(rs)
                for e in range(elem_off[p], elem_off[p + 1]):
                    g = e * n_classes + cl
                    c0, c1, g0, g1 = cand_off[g], cand_off[g + 1], gt_off[g], gt_off[g + 1]
                    code = np.full(c1 - c0, -1)
                    if g1 > g0 and c1 > c0:
                        ov = _iou_rows(cand[c0:c1], gt[g0:g1], dim)
                        for i in range(c1 - c0):
                            if np.isnan(ov[i]).any():
                                code[i] = -2
                            elif ov[i].max() > t:
                                code[i] = int(np.argmax(ov[i]))
                    best = np.full(g1 - g0, -1)
                    for j in range(g1 - g0):
                        for i in range(c1 - c0):
                            if code[i] == j and (best[j] < 0 or _beats(score[c0 + i], score[c0 + best[j]])):
                                best[j] = i
                    for cat in range(3):
                        for i in range(c1 - c0):
                            c = code[i]
                            f = c == -1 if cat == 2 else (c >= 0 and ((best[c] == i) == (cat == 1)))
                            if f:
                                rs.append(score[c0 + i])
                                rm.append((0 if cat == 1 else 1, cl, p, iu))
                    for j in range(g1 - g0):
                        if best[j] < 0:
                            rs.append(0.0)
                            rm.append((2, cl, p, iu))
                if len(rs) == start:
                    rs.append(0.0)
                    rm.append((3, cl, p, iu))
    return np.array(rs, dtype=np.float64), np.array(rm, dtype=np.int32).reshape(-1, 4)


def roi_ap(score, seg, kind, n_seg, thresholds, recall_points):
    """mdt_eval_roi_ap: q [n_seg, n_thresh, n_recall], counts [n_seg, 1 + n_thresh] = (all_p, nd per threshold)"""
    n_thr, n_r = len(thresholds), len(recall_points)
    q = np.zeros((n_seg, n_thr, n_r))
    counts = np.zeros((n_seg, 1 + n_thr), dtype=np.int32)
    counts[:, 0] = np.bincount(seg[(seg >= 0) & ((kind == 0) | (kind == 2))], minlength=n_seg)
    ranked = np.nonzero((seg >= 0) & ((kind == 0) | (kind == 1)) & ~np.isnan(score))[0]
    ranked = ranked[np.argsort(seg[ranked], kind='stable')]          # grouped by segment once, each group in row order
    bounds = np.searchsorted(seg[ranked], np.arange(n_seg + 1))
    for s in range(n_seg):
        idx = ranked[bounds[s]:bounds[s + 1]]
        idx = idx[np.argsort(-score[idx], kind='stable')]
        ss = score[idx]
        tpc = np.cumsum(kind[idx] == 0)
        all_p = int(counts[s, 0])
        for ti, t in enumerate(thresholds):
            nd = int((ss > t).sum())
            counts[s, 1 + ti] = nd
            if nd == 0 or all_p == 0:
                continue
            rc = tpc[:nd] / all_p
            env = np.maximum.accumulate((tpc[:nd] / np.arange(1, nd + 1))[::-1])[::-1]
            at = np.searchsorted(rc, recall_points, side='left')
            q[s, ti] = np.where(at < nd, env[np.minimum(at, nd - 1)], 0.0)
    return q, counts


def patient_counts(score, label, slot, n_slots, members):
    """mdt_eval_patient: per segment (an array of slots) the distinct patient scores in descending order with tps / fps at each"""
    lab = np.full(n_slots, -1)
    mx = np.full(n_slots, -np.inf)
    ok = slot >= 0
    np.maximum.at(lab, slot[ok], label[ok])
    np.maximum.at(mx, slot[ok], score[ok])
    out = []
    for m in members:
        m = m[lab[m] >= 0]
        s, y = mx[m], lab[m]
        u = np.unique(s)[::-1]
        out.append((u, np.array([(y[s >= v] == 1).sum() for v in u], dtype=np.int32),
                    np.array([(y[s >= v] != 1).sum() for v in u], dtype=np.int32)))
    return out


def run_metric_kernels(roi, pat, thresholds):
    """the oracle counterpart of evaluator._run_metric_kernels (same inputs, same result dict)"""
    from medicaldetectiontoolkit_b200.evaluator import RECALL_POINTS
    res = {}
    if roi.n_seg:
        idx = np.concatenate(roi.rows)
        res['q'], res['counts'] = roi_ap(roi.c['pred_score'][idx], np.concatenate(roi.segs), roi.codes[idx], roi.n_seg, thresholds, RECALL_POINTS)
    if pat.members:
        curves = patient_counts(pat.c['pred_score'], pat.c['class_label'], pat.row_slot, max(pat.n_slots, 1), pat.members)
        n_members = sum(m.size for m in pat.members)
        res['thr'] = np.zeros(max(n_members, 1))
        res['tps'] = np.zeros(max(n_members, 1), dtype=np.int32)
        res['fps'] = np.zeros(max(n_members, 1), dtype=np.int32)
        res['n_thr'] = np.array([c[0].size for c in curves], dtype=np.int32)
        off = 0
        for m, (u, tp, fp) in zip(pat.members, curves):
            res['thr'][off:off + u.size], res['tps'][off:off + u.size], res['fps'][off:off + u.size] = u, tp, fp
            off += m.size
    return res


def patch(evaluator_module):
    """run medicaldetectiontoolkit_b200.evaluator on this oracle instead of the kernels (returns an undo function)"""
    saved = evaluator_module.match_rows, evaluator_module._run_metric_kernels
    evaluator_module.match_rows = match_rows
    evaluator_module._run_metric_kernels = run_metric_kernels

    def undo():
        evaluator_module.match_rows, evaluator_module._run_metric_kernels = saved
    return undo
