"""The evaluation kernels (csrc/evaluate.cu) at the sizes real workloads reach, where they take paths the golden cases never do: match groups
wider than a warp (the lane-strided loops and the chunked ballot placement past the first 32 lanes), ROI-AP row counts on both sides of cub's
single-tile radix-sort limits and far beyond them, with exact score ties spread across tiles, and patient segments longer than one pass of
the 256-thread curve loops.  Each C-ABI entry point runs through _guarded (poisoned exact-size outputs and workspaces at three offsets, every
run bit-identical) and is compared with the numpy oracle (oracle/eval_oracle.py, pinned to the reference's goldens by
tests/test_evaluator_cpu.py) with np.array_equal; the Evaluator end to end at epoch scale is compared column by column with the Evaluator
running on the oracle.  Every input is built here from a seed, and every test asserts that its input reaches the regime it is written for.
The check that the ROI tie input tells a stable sort from an unstable one runs on the oracle alone and needs no GPU."""
import copy
import functools
import os
import pickle
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import eval_oracle as O  # noqa: E402
import make_eval_golden as G  # noqa: E402
from _guarded import _run_guarded  # noqa: E402

from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import evaluator as E  # noqa: E402

DEV = "cuda:0"
SORT_TILE_F64 = 256 * 9        # cub's sm_90 single-tile radix sort (CUDA 12.9): the most fp64 keys (the descending score sort) in one tile
SORT_TILE_I32 = 256 * 19       # ... and the most int keys (the segment-id sort)
CURVE_THREADS = 256            # threads of one patient-curve block (kPatThreads)


def _d(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(DEV)


# ------------------------------------------------------------------------------------------------------------------------ matching
CAND_SIZES = (0, 1, 31, 32, 33, 64, 65, 200)
GT_SIZES = (0, 1, 31, 32, 33, 40)
N_CLS = 2


def _box(lo, size, dim):
    hi = lo + size
    return np.array([lo[0], lo[1], hi[0], hi[1]] + ([lo[2], hi[2]] if dim == 3 else []), dtype=np.float64)


def _gts(rs, dim, n_gt, origin):
    """n_gt GT boxes on a grid 40 apart (no two overlap), extents 12..20"""
    return [_box(origin + 40.0 * np.array([j % 8, j // 8, 0][:dim]), rs.uniform(12, 20, dim), dim) for j in range(n_gt)]


def _cands(rs, dim, n_cand, gts, origin, pick):
    """jittered copies of the GTs listed in `pick` (several per GT, from every lane chunk) and boxes that overlap no GT; scores rounded to
    2 decimals, so that a GT's matched candidates often tie"""
    boxes = []
    for _ in range(n_cand):
        if len(pick) and rs.rand() < 0.75:
            g = gts[pick[rs.randint(len(pick))]]
            boxes.append(g + rs.normal(0, rs.choice([0.3, 1.0, 2.0]), size=g.size))
        else:
            boxes.append(_box(origin - 60.0 + rs.uniform(0, 30, dim), rs.uniform(12, 20, dim), dim))
    return boxes, [float(np.round(rs.uniform(0, 1), 2)) for _ in range(n_cand)]


class _Special:
    """one (element, class) group of 200 candidates and 40 GTs with, in lane chunks >= 1: the winner of a double match, an exact score tie
    between chunks (the first index wins), a NaN score after a finite maximum (np.argmax picks the NaN), a zero-volume pair (NaN IoU: no
    row) and a pair whose IoU is exactly one of the match IoUs (strict '>': unmatched there).  Marker scores have 3 decimals, the others 2."""
    DOUBLE = {3: 0.501, 40: 0.901, 70: 0.601}           # copies of GT 0: 40 (chunk 1) has the highest score
    TIE = {2: 0.402, 34: 0.702, 68: 0.702}              # copies of GT 1: 34 (chunk 1) and 68 (chunk 2) tie, 34 wins
    BETWEEN = (50, 0.123)                               # the only copy of GT 2: a TP between 34 and 68, so the TP order shows the tie winner
    NAN = {10: 0.991, 45: np.nan, 80: np.nan}           # copies of GT 3: 45 (chunk 1), the first NaN, wins over the finite maximum at 10
    ZERO_VOL = (90, 0.777)                              # zero-volume copy of the zero-volume GT 39: 0 / 0 IoU
    PAIR = (120, 0.333)                                 # shifted copy of GT 5: its IoU is the last match IoU
    RESERVED = (0, 1, 2, 3, 5, 39)

    def __init__(self, rs, dim, origin):
        gts = _gts(rs, dim, 40, origin)
        gts[39] = _box(gts[39][[0, 1, 4][:dim]], np.zeros(dim), dim)
        pick = [j for j in range(40) if j not in self.RESERVED]
        cands, scores = _cands(rs, dim, 200, gts, origin, pick)
        for gi, table in ((0, self.DOUBLE), (1, self.TIE), (3, self.NAN)):
            for i, s in table.items():
                cands[i], scores[i] = gts[gi].copy(), s
        cands[self.BETWEEN[0]], scores[self.BETWEEN[0]] = gts[2].copy(), self.BETWEEN[1]
        cands[self.ZERO_VOL[0]], scores[self.ZERO_VOL[0]] = gts[39].copy(), self.ZERO_VOL[1]
        shift = np.array([0.25, 0.5, 0.25, 0.5, 0.25, 0.5][:2 * dim])
        cands[self.PAIR[0]], scores[self.PAIR[0]] = gts[5] + shift, self.PAIR[1]
        self.iou = float(O._iou_rows(cands[self.PAIR[0]][None], gts[5][None], dim)[0, 0])
        self.cands, self.scores, self.gts = cands, scores, gts

    def check(self, rs_score, rm, p, ious):
        """the oracle's rows of this group's slots show every construction taking effect"""
        for iu in range(len(ious)):
            sel = (rm[:, 1] == 0) & (rm[:, 2] == p) & (rm[:, 3] == iu)
            tp, fp = list(rs_score[sel & (rm[:, 0] == 0)]), list(rs_score[sel & (rm[:, 0] == 1)])
            assert self.ZERO_VOL[1] not in tp + fp
            assert (self.PAIR[1] in fp) == (iu == len(ious) - 1) and (self.PAIR[1] in tp) == (iu < len(ious) - 1)
            assert 0.901 in tp and 0.501 in fp and 0.601 in fp
            nan_at = [k for k, s in enumerate(tp) if np.isnan(s)]
            assert len(nan_at) == 1 and 0.991 in fp
            assert tp.count(0.702) == 1 and fp.count(0.702) == 1
            assert tp.index(0.702) < nan_at[0] < tp.index(0.123)


@functools.lru_cache(maxsize=None)
def match_case(dim):
    """(flat, ious, special, special patient, group sizes): 700 patients of 1..80 elements (some own nothing at all), mostly small groups,
    every (candidates, GTs) size of CAND_SIZES x GT_SIZES in some group, and the special group"""
    rs = np.random.RandomState(100 + dim)
    n_pat = 700
    n_el = np.where(rs.rand(n_pat) < 0.7, rs.randint(1, 5, n_pat), np.where(rs.rand(n_pat) < 0.85, rs.randint(5, 30, n_pat), 80))
    n_el[:3] = (1, 80, 1)
    elem_off = np.concatenate([[0], np.cumsum(n_el)]).astype(np.int32)
    n_groups = int(elem_off[-1]) * N_CLS
    empty_pat = rs.rand(n_pat) < 0.05
    empty_pat[:3] = (False, False, True)
    sizes = {}
    for g in range(n_groups):
        if not empty_pat[np.searchsorted(elem_off, g // N_CLS, side='right') - 1] and rs.rand() < 0.5:
            sizes[g] = (rs.randint(0, 7), rs.randint(0, 3))
    special_p = 0
    special_g = int(elem_off[special_p]) * N_CLS                 # patient 0's only element, class index 0
    free = [g for g in range(N_CLS * int(elem_off[3]), n_groups) if not empty_pat[np.searchsorted(elem_off, g // N_CLS, side='right') - 1]]
    combos = [(nc, ng) for nc in CAND_SIZES for ng in GT_SIZES]
    for g, combo in zip(rs.choice(free, len(combos), replace=False), combos):
        sizes[int(g)] = combo
    sizes[int(elem_off[1]) * N_CLS + 1] = (200, 40)               # patient 1 (80 elements): a wide group of class index 1 as well
    special = _Special(rs, dim, np.full(dim, 100.0))
    cand, score, gt, cand_n, gt_n = [], [], [], np.zeros(n_groups, np.int64), np.zeros(n_groups, np.int64)
    for g in range(n_groups):
        if g == special_g:
            c, s, t = special.cands, special.scores, special.gts
        else:
            nc, ng = sizes.get(g, (0, 0))
            origin = np.full(dim, 100.0) + rs.uniform(0, 50, dim)
            t = _gts(rs, dim, ng, origin)
            c, s = _cands(rs, dim, nc, t, origin, list(range(ng)))
        cand += c
        score += s
        gt += t
        cand_n[g], gt_n[g] = len(c), len(t)
    flat = (dim, np.array(cand, dtype=np.float64).reshape(-1, 2 * dim), np.array(score, dtype=np.float64),
            np.concatenate([[0], np.cumsum(cand_n)]).astype(np.int32), np.array(gt, dtype=np.float64).reshape(-1, 2 * dim),
            np.concatenate([[0], np.cumsum(gt_n)]).astype(np.int32), elem_off)
    ious = [0.1, 0.25, 0.5, special.iou]
    return flat, ious, special, special_p, (cand_n, gt_n, empty_pat)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [2, 3])
def test_match_wider_than_a_warp(dim):
    flat, ious, special, special_p, (cand_n, gt_n, empty_pat) = match_case(dim)
    _, cand, score, cand_off, gt, gt_off, elem_off = flat
    n_pat, n_iou = elem_off.size - 1, len(ious)
    n_slots = n_iou * N_CLS * n_pat
    # the regime: groups past one lane chunk in both loops, every listed size, thousands of slots, empty patients, 80-element patients
    assert ((cand_n >= 65) & (gt_n >= 33)).any()
    assert {(int(c), int(g)) for c, g in zip(cand_n, gt_n)} >= {(c, g) for c in CAND_SIZES for g in GT_SIZES}
    assert n_slots >= 4000 and (elem_off[1:] - elem_off[:-1]).max() == 80 and empty_pat.sum() >= 10
    assert not np.isin(ious[-1], ious[:-1]) and 0.5 < ious[-1] < 1
    want_s, want_m = O.match_rows(flat, N_CLS, ious)
    special.check(want_s, want_m, special_p, ious)
    tn = want_m[want_m[:, 0] == 3]
    assert set(np.nonzero(empty_pat)[0]) <= set(tn[:, 2])
    max_rows = n_iou * (cand.shape[0] + gt.shape[0] + N_CLS * n_pat)
    lib = L.load()
    ws_b = lib.mdt_eval_match_workspace_bytes(n_slots, cand.shape[0], gt.shape[0], n_iou)
    assert ws_b > 0
    d = [_d(cand, np.float64), _d(score, np.float64), _d(cand_off, np.int32), _d(gt, np.float64), _d(gt_off, np.int32), _d(elem_off, np.int32),
         _d(ious, np.float64)]

    def call(outs, ws):
        return lib.mdt_eval_match(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), cand.shape[0], L.ptr(d[3]), L.ptr(d[4]), gt.shape[0], L.ptr(d[5]), n_pat,
                                  N_CLS, dim, L.ptr(d[6]), n_iou, outs[0], outs[1], outs[2], ws, ws_b, None)
    got = _run_guarded(call, [8 * max_rows, 16 * max_rows, 4], ws_b)
    n = int(got[2].view(torch.int32).item())
    assert n == want_s.size
    assert np.array_equal(got[1].view(torch.int32).reshape(-1, 4)[:n].cpu().numpy(), want_m)
    assert np.array_equal(got[0].view(torch.float64)[:n].cpu().numpy(), want_s, equal_nan=True)


# ------------------------------------------------------------------------------------------------------------------------- ROI AP
# thresholds: min_det_thresh and the scan's, one below zero (so that the +-0.0 and lowest ties are ranked) and one above every score (nd = 0)
ROI_THRESHOLDS = [0.1] + E.SCAN_THRESHOLDS + [-1.0, 2.0]
BIG_SEG = 100_000
ROI_CASES = [          # (rows, segments, recall points)
    (SORT_TILE_F64 - 1, 1, 101), (SORT_TILE_F64, 255, 128), (SORT_TILE_F64 + 1, 256, 1),
    (SORT_TILE_I32 - 1, 257, 101), (SORT_TILE_I32, 1, 128), (SORT_TILE_I32 + 1, 4096, 101),
    (50_000, 256, 128), (50_000, 4096, 1), (400_000, 257, 101), (400_000, 4096, 128)]


@functools.lru_cache(maxsize=None)
def roi_case(n, n_seg):
    """(score, seg, kind) of n rows.  Scores rounded to 2 or 3 decimals with a block of exact 1.0, +0.0 and -0.0 mixed, NaNs, and scores
    equal to each threshold; rows of segment -1 and TN rows.  With n_seg >= 4: segment 1 empty, 2 FN-only, 3 FP-only (all_p = 0); from
    400 000 rows on, segment 0 holds 45 % of them (> 10^5 ranked).  Row order is random, so every tie spans the whole array."""
    rs = np.random.RandomState(n * 7 + n_seg)
    kind = rs.choice(4, n, p=[0.35, 0.45, 0.15, 0.05]).astype(np.int32)
    seg = rs.randint(0, n_seg, n).astype(np.int32)
    if n >= 400_000:
        seg[rs.rand(n) < 0.45] = 0
    if n_seg >= 4:
        seg[seg == 1] = 0
        kind[(seg == 2) & (kind != 3)] = 2
        kind[(seg == 3) & (kind != 3)] = 1
    seg[rs.rand(n) < 0.03] = -1
    score = rs.uniform(0, 1, n)
    score = np.where(rs.rand(n) < 0.5, np.round(score, 2), np.round(score, 3))
    u = rs.rand(n)
    score[u < 0.04] = 1.0
    zero = (u >= 0.04) & (u < 0.07)
    score[zero] = np.where(rs.rand(n) < 0.5, -0.0, 0.0)[zero]
    score[(u >= 0.07) & (u < 0.08)] = np.nan
    at = (u >= 0.08) & (u < 0.11)
    score[at] = np.array(ROI_THRESHOLDS[:-2])[rs.randint(0, len(ROI_THRESHOLDS) - 2, n)][at]
    score[kind >= 2] = 0.0
    return score, seg, kind


def _ranked(score, seg, kind):
    return (seg >= 0) & ((kind == 0) | (kind == 1)) & ~np.isnan(score)


def _check_roi_regime(score, seg, kind, n_seg):
    n = score.size
    ranked = _ranked(score, seg, kind)
    det = (kind == 0) | (kind == 1)
    assert (seg == -1).any() and np.isnan(score[det]).any()
    z = det & (score == 0)
    assert np.signbit(score[z]).any() and (~np.signbit(score[z])).any()
    for t in ROI_THRESHOLDS[:-2]:
        assert (det & (score == t)).any()
    assert np.nanmax(score[det]) < ROI_THRESHOLDS[-1]
    ones = np.nonzero(ranked & (score == 1.0))[0]
    assert ones.size >= 50
    if n >= 2 * SORT_TILE_F64:                                               # exact ties on both sides of a sort-tile boundary
        assert ones.min() < SORT_TILE_F64 <= ones.max()
    if n_seg >= 4:
        present = np.bincount(seg[seg >= 0], minlength=n_seg)
        assert present[1] == 0 and present[2] > 0 and present[3] > 0
        assert (kind[seg == 2] != 0).all() and (kind[seg == 2] != 1).all()
        assert not ((kind[seg == 3] == 0) | (kind[seg == 3] == 2)).any()
    return int(np.bincount(seg[ranked], minlength=n_seg).max())


def test_roi_case_tie_order_changes_the_oracle_ap():
    """reversing the row order of the TP / FP rows tied at 1.0 in the big segment changes the oracle's q: the tie input tells a stable
    sort (ties in row order) from one that is not"""
    score, seg, kind = roi_case(400_000, 4096)
    R = np.linspace(0, 1, 101)
    ties = np.nonzero(_ranked(score, seg, kind) & (seg == 0) & (score == 1.0))[0]
    assert ties.size > 1000 and np.unique(kind[ties]).tolist() == [0, 1]
    flipped = kind.copy()
    flipped[ties] = kind[ties][::-1]
    q, counts = O.roi_ap(score, seg, kind, 4096, ROI_THRESHOLDS, R)
    q2, counts2 = O.roi_ap(score, seg, flipped, 4096, ROI_THRESHOLDS, R)
    assert np.array_equal(counts, counts2)
    assert not np.array_equal(q[0], q2[0]) and np.array_equal(q[1:], q2[1:])


@pytest.mark.gpu
@pytest.mark.parametrize("n,n_seg,n_r", ROI_CASES)
def test_roi_ap_multi_tile(n, n_seg, n_r):
    score, seg, kind = roi_case(n, n_seg)
    biggest = _check_roi_regime(score, seg, kind, n_seg)
    if n >= 400_000:
        assert biggest > BIG_SEG
    R = np.linspace(0, 1, n_r)
    th = ROI_THRESHOLDS
    q, counts = O.roi_ap(score, seg, kind, n_seg, th, R)
    assert (counts[:, -1] == 0).all() and (counts[:, 1:] > 0).any()
    lib = L.load()
    ws_b = lib.mdt_eval_roi_ap_workspace_bytes(n, n_seg)
    assert ws_b > 0
    d = [_d(score, np.float64), _d(seg, np.int32), _d(kind, np.int32), _d(th, np.float64), _d(R, np.float64)]

    def call(outs, ws):
        return lib.mdt_eval_roi_ap(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), n, n_seg, L.ptr(d[3]), len(th), L.ptr(d[4]), n_r, outs[0], outs[1],
                                   ws, ws_b, None)
    got = _run_guarded(call, [8 * n_seg * len(th) * n_r, 4 * n_seg * (1 + len(th))], ws_b)
    assert np.array_equal(got[1].view(torch.int32).cpu().numpy().reshape(counts.shape), counts)
    assert np.array_equal(got[0].view(torch.float64).cpu().numpy().reshape(q.shape), q)


# --------------------------------------------------------------------------------------------------------------------- patient level
PAT_SEG_SIZES = (1, 255, 256, 257, 1000, 3000)


@functools.lru_cache(maxsize=None)
def patient_case():
    """(score, label, slot, n_slots, members): 4 000 slots with 0..4 rows each (about 1 in 8 has none: no patient), scores rounded to 2
    decimals; segments of PAT_SEG_SIZES members, drawn from shared slots (as the folds share the 'all' segment's), the 257-member one from
    slots whose rows all score 0.5"""
    rs = np.random.RandomState(77)
    n_slots = 4000
    equal = np.arange(3600, 3600 + 290)                            # slots whose rows all score 0.5
    per = np.where(rs.rand(n_slots) < 0.12, 0, rs.randint(1, 5, n_slots))
    per[equal] = 2
    slot = np.repeat(np.arange(n_slots, dtype=np.int32), per)
    n = slot.size
    score = np.round(rs.uniform(0, 1, n), 2)
    label = (rs.rand(n) < 0.3).astype(np.int32)
    score[np.isin(slot, equal)] = 0.5
    slot[(rs.rand(n) < 0.05) & ~np.isin(slot, equal)] = -1        # rows of no slot
    order = rs.permutation(n)                                      # rows in no slot order
    score, label, slot = score[order], label[order], slot[order]
    members = [np.array([rs.randint(n_slots)], dtype=np.int32),
               np.sort(rs.choice(3000, 255, replace=False)).astype(np.int32),
               rs.choice(3000, 256, replace=False).astype(np.int32),
               equal[:257].astype(np.int32),
               np.sort(rs.choice(3000, 1000, replace=False)).astype(np.int32),
               np.arange(3000, dtype=np.int32)]
    return score, label, slot, n_slots, members


@pytest.mark.gpu
def test_patient_curves_multi_iteration():
    score, label, slot, n_slots, members = patient_case()
    n = score.size
    have = np.zeros(n_slots, bool)
    have[slot[slot >= 0]] = True
    assert [m.size for m in members] == list(PAT_SEG_SIZES) and max(m.size for m in members) > CURVE_THREADS
    assert all((~have[m]).any() for m in members[4:]) and have[members[3]].all() and have[members[3]].sum() > CURVE_THREADS
    assert np.unique(score[np.isin(slot, members[3])]).tolist() == [0.5] and np.isfinite(score).all()
    assert np.isin(members[4], members[5]).all() and np.isin(members[2], members[5]).all()
    want = O.patient_counts(score, label, slot, n_slots, members)
    assert want[3][0].size == 1 and want[5][0].size > 50
    off = np.concatenate([[0], np.cumsum([m.size for m in members])]).astype(np.int32)
    n_mem = int(off[-1])
    lib = L.load()
    ws_b = lib.mdt_eval_patient_workspace_bytes(n_slots, n_mem)
    d = [_d(score, np.float64), _d(label, np.int32), _d(slot, np.int32), _d(off, np.int32), _d(np.concatenate(members), np.int32)]

    def call(outs, ws):
        return lib.mdt_eval_patient(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), n, n_slots, L.ptr(d[3]), L.ptr(d[4]), n_mem, len(members), outs[0],
                                    outs[1], outs[2], outs[3], ws, ws_b, None)
    got = _run_guarded(call, [8 * n_mem, 4 * n_mem, 4 * n_mem, 4 * len(members)], ws_b)
    n_thr = got[3].view(torch.int32).cpu().numpy()
    thr, tps, fps = (got[i].view(dt).cpu().numpy() for i, dt in ((0, torch.float64), (1, torch.int32), (2, torch.int32)))
    assert np.array_equal(n_thr, [u.size for u, _, _ in want])
    for k, (u, tp, fp) in enumerate(want):
        sl = slice(off[k], off[k] + u.size)
        assert np.array_equal(thr[sl], u) and np.array_equal(tps[sl], tp) and np.array_equal(fps[sl], fp)


# -------------------------------------------------------------------------------------------------------------------- end to end
def _det_score(rs):
    """an fp32 softmax foreground probability widened to fp64: about 1 in 20 saturates at exactly 1.0"""
    z = np.float32(rs.normal(2.0, 8.0))
    return float(np.float32(1) / (np.float32(1) + np.exp(-z, dtype=np.float32)))


def _e2e_element(rs, dim, n_det, n_gt_max=3, extent=128.0):
    boxes = []
    for cl in (1, 2):
        gts = [G._box(rs, dim, extent) for _ in range(rs.randint(0, n_gt_max + 1))]
        boxes += [{'box_coords': g, 'box_type': 'gt', 'box_label': cl} for g in gts]
        for _ in range(n_det() if callable(n_det) else n_det):
            if gts and rs.rand() < 0.4:
                d = gts[rs.randint(len(gts))] + rs.normal(0, rs.choice([0.5, 2.0, 5.0]), size=2 * dim)
            else:
                d = G._box(rs, dim, extent)
            boxes.append({'box_coords': d, 'box_type': 'det', 'box_score': _det_score(rs), 'box_pred_class_id': cl})
    return boxes


def e2e_case(name):
    rs = np.random.RandomState(sum(map(ord, name)))
    if name == 'lidc3d_train_epoch':             # 200 batches of 8 elements, 30 detections per element and class
        res = [[[_e2e_element(rs, 3, 30) for _ in range(8)], ['p%d' % rs.randint(800) for _ in range(8)]] for _ in range(200)]
        return G.base_cf(), 'train', res
    if name == 'test_1000_scan_per_patient':    # 1 000 one-element patients, 50..300 detections per class, three IoUs
        res = [[[_e2e_element(rs, 3, lambda: rs.randint(50, 301))], 'p%04d' % p] for p in range(1000)]
        return G.base_cf(ap_match_ious=[0.1, 0.25, 0.5], per_patient_ap=True, scan_det_thresh=True), 'test', res
    if name == 'val_patient_2d_64':             # 200 patients of 64 slices; about half have GT boxes, in a run of 4..20 slices
        res = []
        for p in range(200):
            lo = rs.randint(0, 44)
            hi = lo + rs.randint(4, 21) if rs.rand() < 0.5 else lo
            res.append([[_e2e_element(rs, 2, lambda: rs.randint(0, 5), n_gt_max=2 if lo <= z < hi else 0) for z in range(64)], 'q%03d' % p])
        return G.base_cf(), 'val_patient', res
    raise KeyError(name)


def _evaluate(cf, mode, res):
    ev = E.Evaluator(cf, G.Logger(), mode)
    np.random.seed(G.RNG_SEED)
    if mode == 'test':
        ev.evaluate_predictions(copy.deepcopy(res))
        stats, mm = ev.return_metrics()
    else:
        stats, mm = ev.evaluate_predictions(copy.deepcopy(res), G.new_monitor_metrics(cf))
    return ev, stats, mm


@pytest.mark.gpu
@pytest.mark.parametrize("name", ['lidc3d_train_epoch', 'test_1000_scan_per_patient', 'val_patient_2d_64'])
def test_evaluator_end_to_end_at_epoch_scale(name):
    cf, mode, res = e2e_case(name)
    ev, stats, mm = _evaluate(cf, mode, res)
    ev_b, stats_b, mm_b = _evaluate(cf, mode, res)
    undo = O.patch(E)
    try:
        ev_o, stats_o, mm_o = _evaluate(cf, mode, res)
    finally:
        undo()
    c = ev.columns
    det = (c['det_type'] == 'det_tp') | (c['det_type'] == 'det_fp')
    n_det = sum(b['box_type'] == 'det' for item in res for el in item[0] for b in el)
    if name == 'lidc3d_train_epoch':
        assert n_det == 96_000 and (c['pred_score'][det] == 1.0).sum() > 1000
    if name == 'test_1000_scan_per_patient':
        assert len({p for p in c['pid']}) == 1000 and cf.per_patient_ap and cf.scan_det_thresh
        assert max(np.unique(c['pid'][c['pred_class'] == cl]).size for cl in (1, 2)) >= 1000
    if name == 'val_patient_2d_64':
        assert len(res) == 200 and all(len(item[0]) == 64 for item in res)
    if mode != 'train':                          # positive and negative patients: the patient-level curves are not degenerate
        assert all(np.isfinite(s['auc']) for s in stats if 'patient' in s['name'])
    for k in c:
        assert np.array_equal(np.asarray(c[k]), np.asarray(ev_o.columns[k])), k
        assert np.array_equal(np.asarray(c[k]), np.asarray(ev_b.columns[k])), k
    assert pickle.dumps(stats) == pickle.dumps(stats_o)
    assert pickle.dumps(stats) == pickle.dumps(stats_b)
    assert pickle.dumps(mm) == pickle.dumps(mm_o)
