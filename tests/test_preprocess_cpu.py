"""LIDC preprocessing on the host against the golden of the reference's own preprocessing.py (tests/golden/make_preprocess_golden.py): the
oracle's restatement bit for bit, the package's pp_patient / preprocess_lidc with a numpy stand-in for the device ops, and the resize
restatement's two interpolation branches against each other."""
import gzip
import os
import pickle

import numpy as np
import pandas as pd
import pytest

import _preprocess_cases as PC
from _preprocess_cases import PO
from medicaldetectiontoolkit_b200 import preprocessing as P
from medicaldetectiontoolkit_b200.configs import make_cf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'preprocess.pkl.gz')


@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return pickle.load(f)


@pytest.fixture(scope='module')
def raw(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('lidc_raw'))
    return root, PC.make_raw_dir(root)


def _oracle_inputs(root, raw_dir, pid):
    """the patient's arrays grouped as the reference groups them, ROI ids and listings sorted"""
    d = os.path.join(raw_dir, pid)
    files = sorted(os.listdir(d))
    chars = pd.read_csv(os.path.join(root, 'characteristics.csv'), sep=';')
    mal = {(r.PatientID, r.NoduleID): r.Malignancy for r in chars.itertuples()}
    rois = []
    for rid in sorted({f.split('.')[0].split('_')[-1] for f in files if f.endswith('.nii.gz')}):
        names = [f for f in files if (rid + '.nii') in f]
        scores = [mal[(pid, int(f.split('_')[2]))] for f in names]
        label = np.mean(scores + [0] * (4 - len(scores)))
        rois.append((names, [PC.npy_reader(os.path.join(d, f)) for f in names], label))
    ct, sp = PC.npy_reader(os.path.join(d, '%s_ct_scan.nrrd' % pid))
    return ct, sp, rois


def _cf(root, raw_dir, pp_dir):
    cf = make_cf(exp='lidc_exp')
    cf.root_dir, cf.raw_data_dir, cf.pp_dir = root, raw_dir, pp_dir
    return cf


def test_cases_cover_the_regimes(golden):
    pats = {pid: (shape, sp) for pid, shape, sp, _ in PC.PATIENTS}
    radii = []
    for pid, (shape, sp) in pats.items():
        out = PO.target_shape(shape, sp, PC.TARGET_SPACING)
        f = np.asarray(shape, float) / np.asarray(out, float)
        radii += [int(4 * max(0, (x - 1) / 2) + 0.5) for x in f]
    assert {1, 2, 3} <= set(radii)
    assert any(PO.target_shape(s, sp, PC.TARGET_SPACING)[2] == s[2] for s, sp in pats.values())     # the 2-D warp branch
    assert golden['suppressed'] and not golden['patients']['LIDC-IDRI-0004']['rois'].any()
    assert golden['patients']['LIDC-IDRI-0004']['meta']['fg_slices'] == []
    assert len(golden['patients']['LIDC-IDRI-0001']['meta']['class_target']) == 3


@pytest.mark.parametrize('pid', [p[0] for p in PC.PATIENTS])
def test_oracle_matches_golden(golden, raw, pid):
    root, raw_dir = raw
    ct, sp, rois = _oracle_inputs(root, raw_dir, pid)
    got = PO.pp_patient(ct, sp, rois, PC.TARGET_SPACING, stats='numpy')
    want = golden['patients'][pid]
    assert got['img'].dtype == np.float32 and np.array_equal(got['img'].view(np.uint32), want['img'].view(np.uint32))
    assert got['rois'].dtype == np.uint8 and np.array_equal(got['rois'], want['rois'])
    assert np.array_equal(got['class_target'], want['meta']['class_target'])
    assert got['fg_slices'] == want['meta']['fg_slices']
    assert want['meta']['spacing'] == sp and want['meta']['pid'] == pid
    assert ''.join(' '.join(s) for s in got['suppressed']) == (golden['suppressed'] if pid == 'LIDC-IDRI-0002' else '')


def test_device_statistics_differ_from_numpys_only_in_the_last_bits(raw):
    root, raw_dir = raw
    for pid, *_ in PC.PATIENTS:
        ct, sp, _ = _oracle_inputs(root, raw_dir, pid)
        x = PO.resample_array(ct, sp, PC.TARGET_SPACING)
        a, m_dev, s_dev = PO.normalize(x, 'device')
        b, m_np, s_np = PO.normalize(x, 'numpy')
        assert s_dev == s_np
        assert abs(float(m_dev) - float(m_np)) <= 2 * np.spacing(abs(m_np))
        assert np.abs(a - b).max() <= 2 * np.spacing(abs(m_np)) / float(s_np) + np.spacing(np.abs(b)).max()


def _compare_dir(golden, pp_dir):
    for pid, want in golden['patients'].items():
        img = np.load(os.path.join(pp_dir, '%s_img.npy' % pid))
        rois = np.load(os.path.join(pp_dir, '%s_rois.npy' % pid))
        assert img.dtype == np.float32 and np.array_equal(img.view(np.uint32), want['img'].view(np.uint32)), pid
        assert rois.dtype == np.uint8 and np.array_equal(rois, want['rois']), pid
        with open(os.path.join(pp_dir, 'meta_info_%s.pickle' % pid), 'rb') as f:
            meta = pickle.load(f)
        assert list(meta) == list(want['meta'])
        assert meta['pid'] == pid and meta['spacing'] == want['meta']['spacing'] and meta['fg_slices'] == want['meta']['fg_slices']
        assert np.array_equal(meta['class_target'], want['meta']['class_target'])
        assert meta['class_target'].dtype == want['meta']['class_target'].dtype
    for name in ('info_df.pickle', 'info_df_bk.pickle'):
        df = pd.read_pickle(os.path.join(pp_dir, name))
        assert list(df.columns) == list(golden['info_df'])
        for c, vals in golden['info_df'].items():
            got = list(df[c])
            assert len(got) == len(vals)
            for g, w in zip(got, vals):
                assert np.array_equal(np.asarray(g), np.asarray(w)), (c, g, w)
    with open(os.path.join(pp_dir, 'suppressed_rois.txt')) as f:
        assert f.read() == golden['suppressed']


def test_package_with_numpy_ops_matches_golden(golden, raw, tmp_path):
    root, raw_dir = raw
    cf = _cf(root, raw_dir, str(tmp_path / 'pp'))
    P.preprocess_lidc(cf, read_image=PC.npy_reader, ops=PC.NumpyOps('numpy'))
    _compare_dir(golden, cf.pp_dir)


def test_resize_branches_agree():
    rs = np.random.RandomState(3)
    for in_shape, out_shape in [((24, 40, 44), (38, 34, 44)), ((9, 30, 7), (4, 61, 7)), ((16, 12, 5), (16, 12, 5)), ((5, 50, 3), (13, 17, 3)),
                                ((40, 33), (17, 70)), ((1, 1, 6), (3, 1, 6))]:
        img = rs.normal(0, 300, in_shape)
        a = PO.resize(img, out_shape, branch='nd')
        b = PO.resize(img, out_shape, branch='warp')
        assert a.shape == b.shape == out_shape
        assert np.abs(a - b).max() <= 1e-12 * np.abs(a).max(), (in_shape, out_shape)


def test_target_shape_and_argument_checks():
    assert P.target_shape((24, 40, 48), (0.9, 0.85, 2.0), (0.7, 0.7, 1.25)) == PO.target_shape((24, 40, 48), (0.9, 0.85, 2.0), (0.7, 0.7, 1.25))
    assert P.target_shape((10, 10, 48), (0.7, 0.7, 1.25), (0.7, 0.7, 1.25)) == [10, 10, 47]     # 48 * 0.7 / 0.7 < 48 in fp64
    assert P.target_shape((2, 2, 2), (0.70049, 0.7, 1.0), (0.7, 0.7, 1.25)) == [1, 2, 2]         # the spacing is rounded to 3 decimals
    with pytest.raises(AssertionError):
        P.target_shape((1, 10, 10), (0.7, 0.7, 1.0), (0.7, 0.7, 1.25))
    for dt in (np.float64, np.int32, np.uint16, bool):
        with pytest.raises(ValueError):
            P.resample_array(np.zeros((4, 4, 4), dt), (1, 1, 1), (0.7, 0.7, 1.25))
    with pytest.raises(ValueError):
        P.resample_array(np.zeros((4, 4), np.int16), (1, 1), (0.7, 0.7))


def test_default_reader_needs_simpleitk():
    try:
        import SimpleITK  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match='SimpleITK'):
            P.sitk_read_image('scan.nrrd')
    else:
        pytest.skip('SimpleITK is installed')


def test_configs_carry_the_preprocessing_attributes():
    cf = make_cf(exp='lidc_exp')
    assert cf.target_spacing == (0.7, 0.7, 1.25)
    assert cf.root_dir is None and cf.raw_data_dir is None and cf.pp_dir is None
    assert not hasattr(make_cf(exp='toy_exp'), 'target_spacing')
