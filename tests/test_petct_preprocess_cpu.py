"""PET-CT preprocessing and the pet_ct PatientBatchIterator on the host: the oracle and the package (with a numpy stand-in for the device
ops) against the golden of the reference's own preprocessing.py (tests/golden/make_petct_preprocess_golden.py), collect_paths, the config
attributes, and the iterator against a restatement from get_patch_crop_coords, edge padding and the seg_rois oracle."""
import gzip
import logging
import os
import pickle

import numpy as np
import pandas as pd
import pytest
from scipy import ndimage

import _petct_preprocess_cases as PC
import _seg_rois_oracle as SRO
from _petct_preprocess_cases import PO
from _loader_cases import NumpyOps as LoaderNumpyOps
from medicaldetectiontoolkit_b200 import data_loader as D
from medicaldetectiontoolkit_b200 import petct_preprocessing as P
from medicaldetectiontoolkit_b200.configs import make_cf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'petct_preprocess.pkl.gz')
PETCT = 'pet_ct_tnm_classification'


@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return pickle.load(f)


@pytest.fixture(scope='module')
def raw(tmp_path_factory):
    return PC.make_raw_dir(str(tmp_path_factory.mktemp('petct_raw')))


def _inputs(path):
    ct, *cg = PC.read_image(os.path.join(path, 'lsa_ct.nii.gz'))
    pet, *pg = PC.read_image(os.path.join(path, 'lsa_pet.nii.gz'))
    rd, h = PC.read_seg(os.path.join(path, 'lsa.seg.nrrd'))
    return ct, cg, pet, pg, rd, h


def _outcome(fn):
    try:
        return tuple(int(v) for v in fn())
    except (ValueError, RecursionError) as e:
        return type(e).__name__


def test_cases_cover_the_regimes(golden):
    z = golden['zcrop']
    assert z['wraps'][0] < 0 and z['empty'] == 'ValueError' and z['never_settles'] == 'RecursionError'
    assert z['past_end'][1] > PC.zcrop_cases()['past_end'][0].shape[0]
    pats = golden['patients']
    assert [p['row']['class_target'] for p in pats.values()] == [['T_primary'], ['T_primary'], []]
    assert pats['TNM_study_a/pat_02']['zcrop'][0] < 0 and pats['TNM_study_a/pat_02']['img'].shape[1] > 0
    assert pats['TNM_study_a/pat_01']['zcrop'][1] > pats['TNM_study_a/pat_01']['img'].shape[1] + pats['TNM_study_a/pat_01']['zcrop'][0]


@pytest.mark.parametrize('name', sorted(PC.zcrop_cases()))
def test_zcrops_oracle_and_package_against_golden(golden, name):
    vol, kw = PC.zcrop_cases()[name]
    assert _outcome(lambda: PO.get_z_crops(vol, 0, **kw)) == golden['zcrop'][name]
    assert _outcome(lambda: P.get_z_crops(vol, 0, ops=PC.NumpyOps(), **kw)) == golden['zcrop'][name]


def test_diagonal_border_needs_8_connectivity():
    """the 4-connected clear_border would keep the square that meets the border diagonally and start the crop ten slices earlier"""
    vol, kw = PC.zcrop_cases()['diagonal_border']
    sl = vol[10] < -600
    lab4, _ = ndimage.label(sl)
    four = sl & ~np.isin(lab4, np.unique(np.concatenate([lab4[0], lab4[-1], lab4[:, 0], lab4[:, -1]])))
    assert ndimage.label(four)[1] == 2 and ndimage.label(PO.clear_border(sl))[1] == 1


def test_oracle_pp_patient_against_golden(golden, raw):
    for rel, _, _, _ in PC.PATIENTS:
        g = golden['patients'][rel]
        img, rois, ct, fg, zc = PO.pp_patient(*_inputs(os.path.join(raw, rel)))
        np.testing.assert_array_equal(img, g['img'])
        np.testing.assert_array_equal(rois, g['rois'])
        assert ct == g['row']['class_target'] and fg == g['row']['fg_slices'] and tuple(int(v) for v in zc) == g['zcrop']


def test_package_preprocess_petct_against_golden(golden, raw, tmp_path):
    cf = make_cf(exp=PETCT)
    cf.raw_data_dir, cf.pp_dir = raw, str(tmp_path / 'pp')
    df = P.preprocess_petct(cf, read_image=PC.read_image, read_seg=PC.read_seg, ops=PC.NumpyOps())
    stored = pd.read_pickle(os.path.join(cf.pp_dir, 'info_df.pickle'))
    assert list(stored.columns) == P.INFO_COLUMNS and list(stored.pid) == [0, 1, 2]
    for pid, (rel, _, _, _) in enumerate(PC.PATIENTS):
        g = golden['patients'][rel]
        img = np.load(os.path.join(cf.pp_dir, '%d_img.npy' % pid))
        rois = np.load(os.path.join(cf.pp_dir, '%d_rois.npy' % pid))
        assert img.dtype == np.float32 and rois.dtype == np.uint8
        np.testing.assert_array_equal(img, g['img'])
        np.testing.assert_array_equal(rois, g['rois'])
        row = stored.iloc[pid]
        assert row.raw_pid == g['row']['raw_pid'] and row.class_target == g['row']['class_target'] and row.fg_slices == g['row']['fg_slices']
    assert len(df) == 3


def test_device_statistics_stay_close(golden, raw):
    """the stand-in with the device's fp64 statistics: each channel within 1e-5 of its largest magnitude in the golden"""
    for rel, _, _, _ in PC.PATIENTS:
        g = golden['patients'][rel]['img']
        img = P.process_patient(*_inputs(os.path.join(raw, rel)), ops=PC.NumpyOps(stats='device'))[0]
        for c in range(2):
            assert np.abs(img[c] - g[c]).max() <= 1e-5 * np.abs(g[c]).max()


def test_collect_paths_sorted_and_filtered(raw):
    paths = P.collect_paths(raw)
    assert paths == sorted(os.path.join(raw, rel) for rel, _, _, _ in PC.PATIENTS)


def test_make_cf_attributes():
    cf = make_cf(exp=PETCT)
    assert cf.root_dir is None and cf.raw_data_dir is None and cf.pp_dir is None


def test_dtype_errors():
    ops = PC.NumpyOps()
    ct, cg, pet, pg, rd, h = (np.zeros((4, 4, 4), np.int16), ((1.0,) * 3, (0.0,) * 3, P.IDENTITY), np.zeros((4, 4, 4), np.float32),
                              ((1.0,) * 3, (0.0,) * 3, P.IDENTITY), np.zeros((4, 4, 4), np.uint8),
                              {'space directions': np.eye(3), 'space origin': np.zeros(3), 'Segment0_Name': 'T_primary'})
    with pytest.raises(ValueError):
        P.process_patient(ct.astype(np.float32), cg, pet, pg, rd, h, ops=ops)
    with pytest.raises(ValueError):
        P.process_patient(ct, cg, pet.astype(np.float64), pg, rd, h, ops=ops)
    with pytest.raises(ValueError):
        P.process_patient(ct, cg, pet, pg, rd.astype(np.int64), h, ops=ops)


# ------------------------------------------------------------------------------------------------------------------- PatientBatchIterator
class IteratorOps(LoaderNumpyOps):
    """the loader's numpy stand-in plus seg_rois in the device op's format"""

    def seg_rois(self, seg, class_target, class_specific):
        first, stats, out = [0], [], np.copy(seg)
        for b in range(seg.shape[0]):
            lab, n = ndimage.label(seg[b, 0] != 0)
            for k in range(1, n + 1):
                ix = np.argwhere(lab == k)
                lo, hi = np.zeros(3, np.int64), np.zeros(3, np.int64)
                lo[:ix.shape[1]], hi[:ix.shape[1]] = ix.min(0), ix.max(0)
                stats.append([len(ix), *lo, *hi])
            first.append(first[-1] + n)
            out[b, 0] = np.where(seg[b, 0] > 0, (class_target[b] + 1) if class_specific else 1, seg[b, 0])
        return np.array(first, np.int32), np.array(stats, np.int32).reshape(-1, 7), out


def make_pp_dir(d, rs):
    """a small preprocessed pet_ct directory: (2, z, y, x) float32 images, binary seg with a few blobs, one patient without foreground"""
    shapes = [(10, 40, 28), (6, 20, 20), (12, 36, 44)]
    rows = []
    for pid, shape in enumerate(shapes):
        img = rs.randn(2, *shape).astype(np.float32)
        seg = np.zeros(shape, np.uint8)
        if pid != 1:
            for _ in range(3):
                z, y, x = (rs.randint(0, s - 3) for s in shape)
                seg[z:z + 3, y:y + rs.randint(2, 6), x:x + rs.randint(2, 6)] = 1
        np.save(os.path.join(d, '%d_img.npy' % pid), img)
        np.save(os.path.join(d, '%d_rois.npy' % pid), seg)
        rows.append({'pid': pid, 'raw_pid': 'p%d' % pid, 'class_target': ['T'] if seg.any() else [],
                     'fg_slices': [np.int64(z) for z in np.flatnonzero(seg.any(axis=(1, 2)))]})
    df = pd.DataFrame(columns=P.INFO_COLUMNS)
    for r in rows:
        df.loc[len(df)] = r
    df.to_pickle(os.path.join(d, 'info_df.pickle'))


def iterator_cf(dim, n3=None, merge=True):
    cf = make_cf('retina_unet', dim, [24, 24, 8][:dim], exp=PETCT)
    cf.n_3D_context, cf.merge_2D_to_3D_preds = n3, merge
    return cf


ITERATOR_CASES = [('3d', 3, None, True), ('2d', 2, None, False), ('2d_merge', 2, None, True), ('2d_context', 2, 1, True)]


def restate(img, seg, cf):
    """the pet_ct patient batch from the rule: edge padding, get_patch_crop_coords tiling and the seg_rois oracle"""
    t = np.array([0 if seg.any() else -1])
    P_ = list(cf.patch_size) + ([1] if cf.dim == 2 else [])
    C, Z, Y, X = img.shape
    shape = [max(s, p) for s, p in zip((Y, X, Z), P_)]
    pad = lambda S, new: ((new - S) // 2, new - S - (new - S) // 2)
    img_p = np.pad(img, [(0, 0), pad(Z, shape[2]), pad(Y, shape[0]), pad(X, shape[1])], mode='edge').transpose(0, 2, 3, 1)
    seg_p = np.pad(seg, [pad(Z, shape[2]), pad(Y, shape[0]), pad(X, shape[1])], mode='edge').transpose(1, 2, 0)
    n3 = cf.n_3D_context

    def chans2d(z):
        if n3 is None:
            return img_p[:, :, :, z]
        return np.stack([img_p[0, :, :, zz] if 0 <= zz < Z else np.zeros_like(img_p[0, :, :, 0]) for zz in range(z - n3, z + n3 + 1)])

    rois = lambda s, dim, tg: SRO.seg_rois(s, [int(v) for v in tg], dim, cf.class_specific_seg_flag)
    p3 = rois(seg_p[None, None], 3, t)
    patched = any(shape[d] > P_[d] for d in range(3))
    out = {'patient_bb_target': p3['bb_target'], 'patient_roi_labels': p3['roi_labels']}
    if cf.dim == 3:
        out.update(seg=p3['seg'], class_target=t, bb_target=p3['bb_target'], roi_labels=p3['roi_labels'], original_img_shape=(1, 1, *shape))
        if not patched:
            out['data'] = img_p[None]
    else:
        s2 = seg_p.transpose(2, 0, 1)[:, None]
        t2 = np.repeat(t, shape[2])
        r2 = rois(s2, 2, t2)
        out.update(seg=r2['seg'], class_target=t2, bb_target=r2['bb_target'], roi_labels=r2['roi_labels'],
                   original_img_shape=(shape[2], C if n3 is None else 2 * n3 + 1, shape[0], shape[1]))
        if not cf.merge_2D_to_3D_preds:
            out.update(patient_bb_target=r2['bb_target'], patient_roi_labels=r2['roi_labels'])
        if not patched:
            out['data'] = np.stack([chans2d(z) for z in range(shape[2])])
    if not patched:
        return out
    coords = D.get_patch_crop_coords(np.zeros(shape, np.uint8), P_)
    if cf.dim == 3:
        data = np.stack([img_p[:, c[0]:c[1], c[2]:c[3], c[4]:c[5]] for c in coords])
        segs = np.stack([seg_p[None, c[0]:c[1], c[2]:c[3], c[4]:c[5]] for c in coords])
    else:
        data = np.stack([chans2d(c[4])[:, c[0]:c[1], c[2]:c[3]] for c in coords])
        segs = np.stack([seg_p[None, c[0]:c[1], c[2]:c[3], c[4]] for c in coords])
    tp = np.repeat(t, len(coords))
    rp = rois(segs, cf.dim, tp)
    out.update(data=data, seg=rp['seg'], class_target=tp, bb_target=rp['bb_target'], roi_labels=rp['roi_labels'], patch_crop_coords=coords)
    return out


def assert_batch_equal(got, want):
    assert sorted(k for k in got if k != 'pid') == sorted(want), (sorted(got), sorted(want))
    for k, v in want.items():
        g = got[k]
        if k in ('bb_target', 'roi_labels', 'patient_bb_target', 'patient_roi_labels'):
            assert len(g) == len(v), k
            for a, b in zip(g, v):
                np.testing.assert_array_equal(np.asarray(a).reshape(-1), np.asarray(b).reshape(-1), err_msg=k)
        elif k == 'original_img_shape':
            assert tuple(g) == tuple(v), k
        else:
            np.testing.assert_array_equal(np.asarray(g), np.asarray(v), err_msg=k)


@pytest.fixture(scope='module')
def pp_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('petct_pp'))
    make_pp_dir(d, np.random.RandomState(7))
    return d


@pytest.mark.parametrize('name,dim,n3,merge', ITERATOR_CASES)
def test_patient_batch_iterator_against_restatement(pp_dir, name, dim, n3, merge):
    cf = iterator_cf(dim, n3, merge)
    cf.pp_data_path = cf.pp_test_data_path = pp_dir
    data = D.load_dataset(cf, logging.getLogger('test'))
    it = D.PatientBatchIterator(data, cf, ops=IteratorOps())
    for pid in range(3):
        got = next(it)
        assert got['pid'] == pid
        assert_batch_equal(got, restate(np.load(os.path.join(pp_dir, '%d_img.npy' % pid)), np.load(os.path.join(pp_dir, '%d_rois.npy' % pid)), cf))
