"""CPU side of the patient bootstrap and the FROC: the FROC oracle (tests/_bootstrap_oracle.py) on hand-computed cases and against a
brute-force sweep, the draw rule, the percentile / NaN rules, and Evaluator.bootstrap / score_bootstrap's host code run on the materialising
oracle: with every multiplicity 1 it gives return_metrics' values bit for bit on every golden case, its chunking changes nothing, and its
argument errors raise ValueError."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bootstrap_oracle as B  # noqa: E402
import make_eval_golden as G  # noqa: E402
from medicaldetectiontoolkit_b200 import evaluator as E  # noqa: E402

NaN = float('nan')


def _froc1(score, kind, lim, threshold=0.1):
    score = np.asarray(score, dtype=np.float64)
    sens, tp, g = B.froc(score, np.zeros(score.size, dtype=np.int64), np.asarray(kind), 1, threshold, lim)
    return sens[0].tolist(), tp[0].tolist(), int(g[0])


def _same(a, b):
    return len(a) == len(b) and all((math.isnan(x) and math.isnan(y)) or x == y for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------------------------- FROC oracle
def test_froc_tp_fp_tie_at_one_score():
    # TP and FP at 0.9: the only operating points are (0, 0) and (1, 1) -- the tie is never split
    sens, tp, g = _froc1([0.9, 0.9, 0.0], [0, 1, 2], [0.5, 1.0])
    assert g == 2 and tp == [0, 1] and sens == [0.0, 0.5]


def test_froc_nan_scores_are_left_out():
    sens, tp, g = _froc1([NaN, 0.8, NaN, 0.7], [0, 1, 1, 0], [0.0, 1.0])
    assert g == 2 and tp == [0, 1] and sens == [0.0, 0.5]


def test_froc_score_at_the_threshold_is_not_a_detection():
    sens, tp, g = _froc1([0.1, 0.5, 0.1000001], [0, 1, 0], [0.0, 1.0])
    assert g == 2 and tp == [0, 1]                     # 0.1 is out; the FP at 0.5 comes first, then the TP at 0.1000001


def test_froc_no_lesion_is_nan():
    sens, tp, g = _froc1([0.9, 0.8], [1, 1], [1.0, 8.0])
    assert g == 0 and tp == [0, 0] and all(math.isnan(s) for s in sens)


def test_froc_only_false_positives():
    sens, tp, g = _froc1([0.9, 0.8, 0.0], [1, 1, 2], [0.5, 8.0])
    assert g == 1 and tp == [0, 0] and sens == [0.0, 0.0]


def test_froc_rate_above_every_fp_count():
    sens, tp, g = _froc1([0.9, 0.8, 0.7, 0.0], [0, 1, 0, 2], [100.0])
    assert g == 3 and tp == [2] and sens == [2 / 3]


def test_froc_fractional_limit():
    # FP counts 1 at 0.8 and 2 at 0.6: a limit of 1.5 allows the point at 0.7 (TP 2, FP 1), not the one at 0.6
    sens, tp, g = _froc1([0.9, 0.8, 0.7, 0.6, 0.5], [0, 1, 0, 1, 0], [0.25 * 6, 0.125 * 6])
    assert g == 3 and tp == [2, 1]


def test_froc_against_a_brute_force_sweep():
    rs = np.random.RandomState(3)
    for _ in range(40):
        n = rs.randint(0, 60)
        score = np.round(rs.uniform(0, 1, n), 1)           # many ties
        score[rs.rand(n) < 0.1] = np.nan
        kind = rs.randint(0, 4, n)
        seg = rs.randint(-1, 3, n)
        lim = np.array([0.125, 0.25, 0.5, 1, 2, 4, 8]) * rs.randint(1, 5)
        sens, tp, g = B.froc(score, seg, kind, 3, 0.1, lim)
        for s in range(3):
            det = (seg == s) & ((kind == 0) | (kind == 1)) & ~np.isnan(score)
            det &= np.where(det, score, -np.inf) > 0.1
            pts = [(0, 0)]
            for v in sorted(set(score[det].tolist())) + [np.inf]:
                sel = det & (score >= v)
                pts.append((int(((kind == 0) & sel).sum()), int(((kind == 1) & sel).sum())))
            want = [max(t for t, f in pts if f <= x) for x in lim]
            assert tp[s].tolist() == want
            gs = int(((seg == s) & ((kind == 0) | (kind == 2))).sum())
            assert g[s] == gs
            assert _same(sens[s].tolist(), [w / gs if gs else NaN for w in want])


# ---------------------------------------------------------------------------------------------------------- draws and intervals
def test_draw_rule_does_not_depend_on_n_resamples():
    a = E.draw_multiplicities(37, 5, 11)
    b = E.draw_multiplicities(37, 20, 11)
    assert np.array_equal(a, b[:5])
    assert (a.sum(axis=1) == 37).all() and a.dtype == np.int32
    for k in range(5):
        assert np.array_equal(a[k], B.draw(11, k, 37))
        assert np.array_equal(a[k], np.bincount(np.random.RandomState([11, k]).randint(0, 37, size=37), minlength=37))
    assert not np.array_equal(E.draw_multiplicities(37, 1, 12)[0], a[0])


def test_interval_is_numpys_percentile_over_the_valid_values():
    v = np.array([0.3, np.nan, 0.1, 0.9, 0.5, np.nan, 0.7])
    lo, hi, n = E.bootstrap_interval(v, 0.1)
    want = np.percentile([0.3, 0.1, 0.9, 0.5, 0.7], [5, 95])
    assert (lo, hi, n) == (want[0], want[1], 5)
    assert E.bootstrap_interval(np.array([0.4]), 0.05) == (0.4, 0.4, 1)
    lo, hi, n = E.bootstrap_interval(np.array([np.nan, np.nan]), 0.05)
    assert math.isnan(lo) and math.isnan(hi) and n == 0
    lo, hi, n = E.bootstrap_interval(np.zeros(0), 0.05)
    assert math.isnan(lo) and n == 0


# ------------------------------------------------------------------------------------------------- the materialising oracle
def test_materialise_keeps_copies_in_place():
    idx, copy = B.materialise(5, np.array([1, 0, 1, 2, 0]), np.array([2, 0, 3]))
    assert idx.tolist() == [1, 1, 3, 3, 3, 4, 4] and copy.tolist() == [0, 1, 0, 1, 2, 0, 1]


# ------------------------------------------------------------------------------- Evaluator.bootstrap's host code on the oracle
@pytest.fixture
def on_oracle():
    undo = B.patch(E)
    yield
    undo()


def _evaluator(name):
    ev, _ = G.run_case(E, name)
    ev.cf.per_patient_ap = False                      # the bootstrap's ROI AP is always over the IoU segments
    ev.cf.scan_det_thresh = False
    return ev


@pytest.mark.parametrize("name", G.CASES)
def test_point_estimates_equal_return_metrics(name, on_oracle):
    ev = _evaluator(name)
    want, _ = ev.return_metrics(None if ev.mode == 'test' else G.new_monitor_metrics(ev.cf))
    got = ev.bootstrap(n_resamples=0)
    assert [g['name'] for g in got] == [w['name'] for w in want]
    for g, w in zip(got, want):
        assert _same([g['ap']['value']], [w['ap']])
        if 'patient' in g['name']:
            assert _same([g['auc']['value']], [w['auc']])
        assert g['ap']['n_valid'] == 0


def test_chunking_and_reruns_change_nothing(on_oracle, monkeypatch):
    ev = _evaluator('test_plain')
    a = ev.bootstrap(n_resamples=6, seed=4)
    va = ev.bootstrap_values
    monkeypatch.setattr(E, 'BOOTSTRAP_CHUNK_BYTES', 1)
    b = ev.bootstrap(n_resamples=6, seed=4)
    assert repr(a) == repr(b)
    for name in va:
        assert repr(va[name]) == repr(ev.bootstrap_values[name])
    c = ev.bootstrap(n_resamples=3, seed=4)           # resample b does not depend on n_resamples
    assert np.array_equal(ev.bootstrap_values['average_foreground_roi']['ap'], va['average_foreground_roi']['ap'][:3], equal_nan=True)
    assert c[0]['ap']['value'] == a[0]['ap']['value']


def test_froc_entries(on_oracle):
    ev = _evaluator('test_plain')
    st = ev.bootstrap(n_resamples=4, fps_per_scan=(0.5, 2))
    rois = [s for s in st if ' rois ' in s['name']]
    assert rois and all(set(s['froc']) == {0.1, 0.25, 0.5} for s in rois)
    for s in rois:
        for iou, f in s['froc'].items():
            assert len(f['sens']) == 2 and s['fps_per_scan'] == (0.5, 2.0)
            raw = ev.bootstrap_values[s['name']]['froc'][iou]
            assert raw['sens'].shape == (4, 2) and raw['cpm'].shape == (4,)
            assert _same(raw['cpm'].tolist(), np.mean(raw['sens'], axis=1).tolist())
            assert _same([f['cpm']['value']], [np.mean([x['value'] for x in f['sens']])])


@pytest.mark.parametrize("kw", [dict(n_resamples=-1), dict(n_resamples=1.5), dict(alpha=0.0), dict(alpha=1.0), dict(alpha=NaN),
                                dict(fps_per_scan=(0.5, 0.0)), dict(fps_per_scan=(1, np.inf)), dict(fps_per_scan=(-1,)),
                                dict(fps_per_scan=())])
def test_bad_arguments_raise(kw, on_oracle):
    ev = _evaluator('edges')
    with pytest.raises(ValueError):
        ev.bootstrap(**kw)


def test_no_rows_raise():
    ev = E.Evaluator(G.base_cf(), G.Logger(), 'test')
    with pytest.raises(ValueError):
        ev.bootstrap()


def test_score_bootstrap_text_matches_results_txt(tmp_path, on_oracle):
    pytest.importorskip('pandas')
    _check_score_bootstrap_text(tmp_path)


def _check_score_bootstrap_text(tmp_path):
    """score_test_df then score_bootstrap on the same rows: each point estimate printed in results_bootstrap.txt equals results.txt's"""
    cf, mode, res = G.case_inputs('fold0')
    cf.exp_dir = str(tmp_path)
    cf.n_cv_splits = 9
    ev = E.Evaluator(cf, G.Logger(), mode)
    ev.evaluate_predictions(res)
    ev.score_test_df()
    ev.score_bootstrap(n_resamples=5, seed=1)
    want = {}
    for ln in open(os.path.join(cf.exp_dir, 'results.txt')):
        p = ln.split()
        if p and p[0] == 'AUC':
            want[' '.join(p[4:])] = (p[1], p[3])
    got = {}
    for ln in open(os.path.join(cf.exp_dir, 'results_bootstrap.txt')):
        p = ln.split()
        if p and p[0] in ('AUC', 'AP') and 'iou' not in p:
            got.setdefault(' '.join(p[6:]), {})[p[0]] = p[1]
            assert p[4] == '(n' and p[5] == '5)'
    assert set(got) == set(want)
    for name, (auc, ap) in want.items():
        assert got[name]['AP'] == ap
        if 'patient' in name:
            assert got[name]['AUC'] == auc
    text = open(os.path.join(cf.exp_dir, 'results_bootstrap.txt')).read()
    assert 'CPM ' in text and 'FROC@0.125 ' in text
