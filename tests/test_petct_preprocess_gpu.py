"""csrc/petct_preprocess.cu, petct_preprocessing.py and the pet_ct PatientBatchIterator on the GPU: every entry point through poisoned
exact-size buffers against oracle/petct_preprocess_oracle.py, preprocess_petct end to end against the golden of the reference's own
preprocessing.py, a CT at a real size, and the written directory feeding training, the patient iterator, Predictor.predict_test_set and the
Evaluator."""
import ctypes
import gzip
import hashlib
import logging
import os
import pickle

import numpy as np
import pytest
import torch

import _petct_preprocess_cases as PC
import test_petct_preprocess_cpu as CPU
from _petct_preprocess_cases import PO
from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import data_loader as D
from medicaldetectiontoolkit_b200 import petct_preprocessing as P
from medicaldetectiontoolkit_b200.configs import make_cf

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
GOLDEN = CPU.GOLDEN
PETCT = CPU.PETCT
_DT = {np.dtype(np.uint8): 0, np.dtype(np.int16): 4, np.dtype(np.float32): 2}


def _poisoned(shape, dtype):
    """an exact-size device buffer of `dtype` with every byte 0xFF"""
    t = torch.from_numpy(np.empty(0, dtype)).dtype
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    return torch.full((n,), 0xFF, dtype=torch.uint8, device=DEV).view(t).view(tuple(shape))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------------------------------------------------------- resample
def _geometries():
    """(name, source array, source grid, output grid)"""
    rs = np.random.RandomState(3)
    ct = rs.randint(-1500, 2000, (30, 40, 44)).astype(np.int16)
    g_ct = P.Grid.of(ct.shape, (0.7, 0.8, 2.0), (-15.0, 17.0, -30.0), PC.FLIP_Y)
    new = P.new_ct_grid(g_ct)
    pet = (rs.rand(9, 8, 9) * 6).astype(np.float32)
    g_pet = P.Grid.of(pet.shape, (4.0, 4.0, 4.0), (-16.0, -16.0, -32.0), P.IDENTITY)
    seg = np.zeros((24, 40, 40), np.uint8)
    seg[5:15, 10:30, 8:25] = 1
    seg[3, 3, 3] = 1
    g_seg = P.Grid.of(seg.shape, (0.6, 0.6, 2.5), (-12.0, -12.0, -25.0), P.IDENTITY)
    rot = (0.0, 1.0, 0.0, -1.0, 0.0, 0.0, 0.0, 0.0, -1.0)     # a rotation with a flip: every input axis maps to another output axis
    g_rot = P.Grid((37, 29, 11), (-14.0, 15.0, 12.0), (1.1, 0.9, 2.7), rot)
    return [('ct_onto_new_grid', ct, g_ct, new), ('pet_onto_ct', pet, g_pet, new), ('seg_onto_ct', seg, g_seg, new),
            ('ct_onto_rotated', ct, g_ct, g_rot), ('pet_onto_rotated', pet, g_pet, g_rot), ('seg_onto_rotated', seg, g_seg, g_rot)]


def _boundary_voxels(src, in_grid, out_grid):
    """output voxels whose interpolated fp64 value lies within 1e-9 of an integer (a truncation boundary)"""
    v = PO.resample(src, in_grid.as_dict(), out_grid.as_dict(), np.float64)
    return np.abs(v - np.round(v)) < 1e-9


@pytest.mark.parametrize('name', [g[0] for g in _geometries()])
@pytest.mark.parametrize('out_dt', [np.uint8, np.int16, np.float32])
def test_resample_matches_oracle(name, out_dt):
    _, src, gi, go = [g for g in _geometries() if g[0] == name][0]
    lib = L.load()
    out = _poisoned(go.shape, out_dt)
    n0 = lib.mdt_launch_count()
    assert lib.mdt_petct_resample(_DT[src.dtype], L.ptr(_dev(src)), ctypes.byref(gi.c_struct()), _DT[np.dtype(out_dt)], L.ptr(out),
                                  ctypes.byref(go.c_struct()), L.stream_ptr()) == 0
    assert lib.mdt_launch_count() == n0 + 1
    got = out.cpu().numpy()
    want = PO.resample(src, gi.as_dict(), go.as_dict(), out_dt)
    if np.dtype(out_dt) == np.float32:
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    else:
        diff = got != want
        assert not (diff & ~_boundary_voxels(src, gi, go)).any()
    if name.startswith('seg') and np.dtype(out_dt) == np.uint8:                 # a binary map stays binary
        assert set(np.unique(got).tolist()) == {0, 1}


def test_resample_rejects_bad_arguments():
    lib = L.load()
    g = P.Grid((2, 2, 2), (0, 0, 0), (1, 1, 1)).c_struct()
    bad = P.Grid((2, 2, 2), (0, 0, 0), (1, 1, 1)).c_struct()
    bad.spacing[1] = 0.0
    s = torch.zeros(8, dtype=torch.int16, device=DEV)
    o = torch.zeros(8, dtype=torch.float32, device=DEV)
    n0 = lib.mdt_launch_count()
    for args in [(3, g, 2, g), (4, g, 3, g), (4, bad, 2, g), (4, g, 2, bad)]:
        assert lib.mdt_petct_resample(args[0], L.ptr(s), ctypes.byref(args[1]), args[2], L.ptr(o), ctypes.byref(args[3]), L.stream_ptr()) == -1
    assert lib.mdt_petct_resample(4, None, ctypes.byref(g), 2, L.ptr(o), ctypes.byref(g), L.stream_ptr()) == -1
    assert lib.mdt_launch_count() == n0
    with pytest.raises(ValueError):
        P.CudaOps(DEV).resample(torch.zeros((2, 2, 2), dtype=torch.float64, device=DEV), P.Grid((2, 2, 2), (0, 0, 0), (1, 1, 1)),
                                P.Grid((2, 2, 2), (0, 0, 0), (1, 1, 1)), np.float32)


# ------------------------------------------------------------------------------------------------------------------- segment merge
@pytest.mark.parametrize('fortran', [False, True])
@pytest.mark.parametrize('dt', [np.uint8, np.int16, np.float32])
def test_seg_merge_matches_oracle(fortran, dt):
    rs = np.random.RandomState(5)
    rd = rs.randint(0, 3, (5, 37, 29, 11)).astype(dt)
    rd = np.asfortranarray(rd) if fortran else rd
    labels = ['T_primary', 'N_inflammation', 'N_1', 'T_other', 'M1']
    sel = [l not in P.BACKGROUND_CATEGORIES for l in labels]
    lib = L.load()
    out = _poisoned((11, 29, 37), np.uint8)
    base = rd if rd.flags.c_contiguous else rd.T
    strides = (ctypes.c_longlong * 4)(*[s // rd.itemsize for s in rd.strides])
    assert lib.mdt_petct_seg_merge(_DT[np.dtype(dt)], L.ptr(_dev(base)), 5, 37, 29, 11, strides, (ctypes.c_ubyte * 5)(*sel), L.ptr(out),
                                   L.stream_ptr()) == 0
    np.testing.assert_array_equal(out.cpu().numpy(), PO.merge_segments(rd, labels))
    np.testing.assert_array_equal(P.CudaOps(DEV).seg_merge(rd, sel).cpu().numpy(), PO.merge_segments(rd, labels))


def test_seg_merge_rejects_bad_arguments():
    lib = L.load()
    s = torch.zeros(8, dtype=torch.uint8, device=DEV)
    st = (ctypes.c_longlong * 4)(8, 4, 2, 1)
    sel = (ctypes.c_ubyte * 300)()
    n0 = lib.mdt_launch_count()
    assert lib.mdt_petct_seg_merge(3, L.ptr(s), 1, 2, 2, 2, st, sel, L.ptr(s), L.stream_ptr()) == -1
    assert lib.mdt_petct_seg_merge(0, L.ptr(s), 0, 2, 2, 2, st, sel, L.ptr(s), L.stream_ptr()) == -1
    assert lib.mdt_petct_seg_merge(0, L.ptr(s), 300, 2, 2, 2, st, sel, L.ptr(s), L.stream_ptr()) == -3
    neg = (ctypes.c_longlong * 4)(8, -4, 2, 1)
    assert lib.mdt_petct_seg_merge(0, L.ptr(s), 1, 2, 2, 2, neg, sel, L.ptr(s), L.stream_ptr()) == -1
    assert lib.mdt_launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------- body components
def _components(vol):
    lib = L.load()
    Z, Y, X = vol.shape
    cap = lib.mdt_petct_body_components_capacity(Z, Y, X)
    assert cap == Z * ((Y * X + 1) // 2)
    ws_bytes = lib.mdt_petct_body_components_workspace_bytes(Z, Y, X)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    label, first, stats = _poisoned((Z, Y, X), np.int32), _poisoned((Z + 1,), np.int32), _poisoned((cap, 3), np.int64)
    assert lib.mdt_petct_body_components(_DT[vol.dtype], L.ptr(_dev(vol)), Z, Y, X, L.ptr(label), L.ptr(first), L.ptr(stats), cap, L.ptr(ws), ws_bytes,
                                         L.stream_ptr()) == 0
    first = first.cpu().numpy()
    return label, first, stats[:first[-1]].cpu().numpy(), (first, stats)


def _zcrop_volumes():
    vols = {k: v for k, (v, _) in PC.zcrop_cases().items()}
    rs = np.random.RandomState(11)
    vols['noise'] = np.where(rs.rand(9, 67, 131) < 0.55, -1000, 0).astype(np.int16)          # many small components, several per warp
    vols['float'] = np.where(rs.rand(5, 40, 33) < 0.6, -700.5, -599.5).astype(np.float32)
    return vols


@pytest.mark.parametrize('name', sorted(_zcrop_volumes()))
def test_body_components_match_oracle(name):
    vol = _zcrop_volumes()[name]
    _, first, stats, dev = _components(vol)
    wf, ws = PO.body_components(vol)
    np.testing.assert_array_equal(first, wf)
    np.testing.assert_array_equal(stats, ws)
    Z, Y, X = vol.shape
    lib = L.load()
    for min_pix, n_comps, rad_crit in [(20, 2, 200), (0, 1, 1e9), (24, 1, 100), (25, 2, 81), (-5, 3, 0)]:
        flags = _poisoned((Z,), np.uint8)
        assert lib.mdt_petct_zcrop_criterion(L.ptr(_dev(first.astype(np.int32))), L.ptr(dev[1]), Z, Y, X, min_pix, n_comps, float(rad_crit),
                                             L.ptr(flags), L.stream_ptr()) == 0
        np.testing.assert_array_equal(flags.cpu().numpy() != 0, PO.zcrop_flags(wf, ws, Y, X, min_pix, n_comps, rad_crit))


@pytest.mark.parametrize('name', sorted(PC.zcrop_cases()))
def test_get_z_crops_matches_golden(golden, name):
    vol, kw = PC.zcrop_cases()[name]
    assert CPU._outcome(lambda: P.get_z_crops(vol, 0, **kw)) == golden['zcrop'][name]
    if name == 'settled':
        assert CPU._outcome(lambda: P.get_z_crops(_dev(vol), 0, **kw)) == golden['zcrop'][name]


def test_body_components_reject_bad_arguments():
    lib = L.load()
    s = torch.zeros(8, dtype=torch.int16, device=DEV)
    n0 = lib.mdt_launch_count()
    assert lib.mdt_petct_body_components_capacity(0, 2, 2) == 0 and lib.mdt_petct_body_components_workspace_bytes(2, 2, 0) == 0
    assert lib.mdt_petct_body_components_capacity(2048, 1024, 1024) == 0
    ws = lib.mdt_petct_body_components_workspace_bytes(2, 2, 2)
    w = torch.zeros(ws, dtype=torch.uint8, device=DEV)
    assert lib.mdt_petct_body_components(3, L.ptr(s), 2, 2, 2, L.ptr(s), L.ptr(s), L.ptr(s), 4, L.ptr(w), ws, L.stream_ptr()) == -1
    assert lib.mdt_petct_body_components(4, L.ptr(s), 2, 2, 2, L.ptr(s), L.ptr(s), L.ptr(s), 3, L.ptr(w), ws, L.stream_ptr()) == -1
    assert lib.mdt_petct_body_components(4, L.ptr(s), 2, 2, 2, L.ptr(s), L.ptr(s), L.ptr(s), 4, L.ptr(w), ws - 1, L.stream_ptr()) == -2
    assert lib.mdt_petct_zcrop_criterion(None, L.ptr(s), 2, 2, 2, 0, 1, 1.0, L.ptr(s), L.stream_ptr()) == -1
    assert lib.mdt_launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------- normalisation
def _ulps(got, want):
    return np.abs(got.astype(np.float64) - want.astype(np.float64)) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


@pytest.mark.parametrize('n', [1, 255, 1025, 262144 + 77])
def test_normalize_matches_oracle(n):
    rs = np.random.RandomState(n)
    ct = rs.randint(-2000, 2000, n).astype(np.int16)
    pet = (rs.gamma(2.0, 1.5, n)).astype(np.float32)
    lib = L.load()
    out, stats = _poisoned((2, n), np.float32), _poisoned((4,), np.float64)
    ws_bytes = lib.mdt_petct_normalize_workspace_bytes(n)
    assert ws_bytes == 16 * 1024
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    assert lib.mdt_petct_normalize(L.ptr(_dev(ct)), L.ptr(_dev(pet)), n, L.ptr(out), L.ptr(stats), L.ptr(ws), ws_bytes, L.stream_ptr()) == 0
    got = out.cpu().numpy()
    want = PO.normalize_device(ct, pet)
    if n == 1:
        assert np.isnan(got).all() and np.isnan(want).all()
        return
    assert _ulps(got, want).max() <= 1.0
    ref = PO.normalize(ct, pet)
    for c in range(2):
        assert np.abs(got[c] - ref[c]).max() <= 1e-5 * np.abs(ref[c]).max()


def test_normalize_rejects_bad_arguments():
    lib = L.load()
    s = torch.zeros(8, dtype=torch.float32, device=DEV)
    n0 = lib.mdt_launch_count()
    assert lib.mdt_petct_normalize_workspace_bytes(0) == 0
    assert lib.mdt_petct_normalize(L.ptr(s), L.ptr(s), 0, L.ptr(s), L.ptr(s), L.ptr(s), 32, L.stream_ptr()) == -1
    assert lib.mdt_petct_normalize(L.ptr(s), L.ptr(s), 8, L.ptr(s), L.ptr(s), L.ptr(s), 16 * 1024 - 1, L.stream_ptr()) == -2
    assert lib.mdt_launch_count() == n0
    with pytest.raises(ValueError):
        P.CudaOps(DEV).normalize(torch.zeros(4, dtype=torch.float32, device=DEV), torch.zeros(4, dtype=torch.float32, device=DEV))


# ------------------------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return pickle.load(f)


@pytest.fixture(scope='module')
def pp(tmp_path_factory):
    raw = PC.make_raw_dir(str(tmp_path_factory.mktemp('petct_raw')))
    out = []
    for k in range(2):
        cf = make_cf(exp=PETCT)
        cf.raw_data_dir, cf.pp_dir = raw, str(tmp_path_factory.mktemp('petct_pp%d' % k))
        P.preprocess_petct(cf, read_image=PC.read_image, read_seg=PC.read_seg)
        out.append(cf.pp_dir)
    return raw, out


def test_preprocess_petct_matches_golden(golden, pp):
    import pandas as pd
    raw, (pp_dir, _) = pp
    df = pd.read_pickle(os.path.join(pp_dir, 'info_df.pickle'))
    for pid, (rel, _, _, _) in enumerate(PC.PATIENTS):
        g = golden['patients'][rel]
        img = np.load(os.path.join(pp_dir, '%d_img.npy' % pid))
        rois = np.load(os.path.join(pp_dir, '%d_rois.npy' % pid))
        assert img.shape == g['img'].shape and img.dtype == np.float32
        np.testing.assert_array_equal(rois, g['rois'])
        row = df.iloc[pid]
        assert row.pid == pid and row.raw_pid == g['row']['raw_pid'] and row.class_target == g['row']['class_target']
        assert row.fg_slices == g['row']['fg_slices']
        for c in range(2):
            assert np.abs(img[c] - g['img'][c]).max() <= 1e-5 * np.abs(g['img'][c]).max()
        # the z-crop of the resampled CT, and the CT channel within 1 ulp of the device-statistics restatement
        ct, cg, pet, pg, rd, h = CPU._inputs(os.path.join(raw, rel))
        want = P.process_patient(ct, cg, pet, pg, rd, h, ops=PC.NumpyOps(stats='device'))[0]
        assert _ulps(img, want).max() <= 1.0
        x_grid = P.Grid.of(ct.shape, *cg)
        new = P.new_ct_grid(x_grid)
        xi = PO.resample(ct, x_grid.as_dict(), new.as_dict(), np.int16) if new is not None else ct
        assert tuple(int(v) for v in P.get_z_crops(xi, pid)) == g['zcrop']


def test_preprocess_petct_is_reproducible(pp):
    _, (a, b) = pp
    digest = lambda d: {f: hashlib.sha256(open(os.path.join(d, f), 'rb').read()).hexdigest() for f in sorted(os.listdir(d)) if f.endswith('.npy')}
    assert digest(a) == digest(b)
    import pandas as pd
    assert pd.read_pickle(os.path.join(a, 'info_df.pickle')).equals(pd.read_pickle(os.path.join(b, 'info_df.pickle')))


def test_ct_at_benchmark_geometry():
    """a 512 x 512 x 300 int16 CT at (0.7, 0.7, 2.0) mm onto the new grid, a few output slices against the oracle"""
    rs = np.random.RandomState(9)
    ct = rs.randint(-1100, 1500, (300, 512, 512)).astype(np.int16)
    gi = P.Grid.of(ct.shape, (0.7, 0.7, 2.0), (-179.0, -179.0, -300.0), P.IDENTITY)
    go = P.new_ct_grid(gi)
    got = P.CudaOps(DEV).resample(_dev(ct), gi, go, np.int16).cpu().numpy()
    assert got.shape == go.shape == (183, 367, 367)
    for z in (0, 1, 91, 182):
        sub = P.Grid((go.size[0], go.size[1], 1), (go.origin[0], go.origin[1], go.origin[2] + z * go.spacing[2]), go.spacing, go.direction)
        want = PO.resample(ct, gi.as_dict(), sub.as_dict(), np.int16)[0]
        diff = got[z] != want
        assert not (diff & ~_boundary_voxels(ct, gi, sub)[0]).any()


class _Log(object):
    def info(self, *a, **k):
        pass

    warning = info


def _cf(dim, pp_dir, exp_dir):
    cf = make_cf('retina_unet', dim, [64, 64, 16][:dim], exp=PETCT)
    cf.pre_crop_size = [72, 72, 20][:dim]
    cf.batch_size = 2
    cf.merge_2D_to_3D_preds = dim == 2          # 3D predictions are already cubes
    cf.pp_data_path = cf.pp_test_data_path = pp_dir
    cf.exp_dir = cf.fold_dir = exp_dir
    cf.n_cv_splits = 3
    for k, v in dict(test_aug=False, merge_3D_iou=0.1, return_masks_in_test=False, wcs_iou=1e-5, fold=0, test_n_epochs=1, folds=[0]).items():
        setattr(cf, k, v)
    return cf


@pytest.mark.parametrize('dim', [3, 2])
def test_preprocessed_directory_feeds_training_prediction_and_evaluation(pp, tmp_path, dim):
    from medicaldetectiontoolkit_b200 import evaluator, predictor, retina_unet
    _, (pp_dir, _) = pp
    cf = _cf(dim, pp_dir, str(tmp_path))
    gens = D.get_train_generators(cf, _Log())
    torch.manual_seed(0)
    net = retina_unet.net(cf, None).to(DEV)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    res = net.train_forward(next(gens['train']))
    opt.zero_grad()
    res['torch_loss'].backward()
    opt.step()
    assert np.isfinite(res['monitor_values']['loss'])
    os.makedirs(os.path.join(str(tmp_path), '1_best_checkpoint'))
    torch.save(net.state_dict(), os.path.join(str(tmp_path), '1_best_checkpoint', 'params.pth'))
    np.save(os.path.join(str(tmp_path), 'epoch_ranking.npy'), np.array([1]))
    gen = D.get_test_generator(cf, _Log())
    assert gen['n_test'] == 3
    results = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(gen)
    assert sorted(pid for _, pid in results) == [0, 1, 2]
    ev = evaluator.Evaluator(cf, _Log(), mode='test')
    ev.evaluate_predictions(results)
    ev.return_metrics()


@pytest.mark.parametrize('name,dim,n3,merge', CPU.ITERATOR_CASES)
def test_patient_batch_iterator_on_gpu_matches_restatement(tmp_path, name, dim, n3, merge):
    CPU.make_pp_dir(str(tmp_path), np.random.RandomState(7))
    cf = CPU.iterator_cf(dim, n3, merge)
    cf.pp_data_path = cf.pp_test_data_path = str(tmp_path)
    it = D.PatientBatchIterator(D.load_dataset(cf, logging.getLogger('test')), cf)
    for pid in range(3):
        got = next(it)
        CPU.assert_batch_equal(got, CPU.restate(np.load(str(tmp_path / ('%d_img.npy' % pid))), np.load(str(tmp_path / ('%d_rois.npy' % pid))), cf))
