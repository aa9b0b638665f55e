"""csrc/preprocess.cu and preprocessing.py on the GPU: each entry point through guarded, poisoned exact-size buffers against
oracle/preprocess_oracle.py, the resample at a real LIDC size against a point-wise fp64 evaluation, and preprocess_lidc end to end
against the golden of the reference's own preprocessing.py, feeding the data loader, a train step and Predictor.predict_test_set."""
import ctypes
import gzip
import os
import pickle

import numpy as np
import pytest
import torch

import _preprocess_cases as PC
from _guarded import DEV, OFFSETS, POISON, _Guarded, _run_guarded
from _preprocess_cases import PO
from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import preprocessing as P

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'preprocess.pkl.gz')
_DT = {np.uint8: 0, np.int16: 4, np.float32: 2}


def _i3(s):
    return (ctypes.c_int * 3)(*[int(v) for v in s])


def _ulps(got, want):
    """|got - want| in units of want's fp32 ulp"""
    return np.abs(got.astype(np.float64) - want.astype(np.float64)) / np.spacing(np.abs(want)).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------- resample
RESAMPLE_CASES = [
    ((8, 9, 10), (13, 17, 19), np.uint8),           # up on every axis
    ((24, 40, 48), (9, 22, 34), np.int16),          # down on every axis, radii 3 / 2 / 1
    ((20, 33, 17), (31, 20, 17), np.float32),       # mixed, last axis unchanged (skimage's warp branch)
    ((37, 65, 129), (50, 41, 200), np.int16),       # extents that are no multiple of any block
    ((5, 6, 7), (1, 6, 7), np.float32),             # single-voxel-thick output
    ((7, 1, 9), (3, 1, 4), np.uint8),
    ((1, 1, 1), (2, 3, 4), np.int16),
    ((64, 5, 6), (3, 5, 6), np.float32),            # factor 21: radius 41
]


def _source(shape, dt, seed):
    rs = np.random.RandomState(seed)
    if dt == np.uint8:
        return (rs.rand(*shape) < 0.4).astype(np.uint8) * rs.randint(1, 3, shape).astype(np.uint8)
    if dt == np.int16:
        return rs.randint(-1500, 3000, shape).astype(np.int16)
    return (rs.normal(0, 400, shape)).astype(np.float32)


@pytest.mark.parametrize('in_shape,out_shape,dt', RESAMPLE_CASES)
def test_resample_matches_oracle(in_shape, out_shape, dt):
    src = _source(in_shape, dt, sum(in_shape) + sum(out_shape))
    want = PO.resize(src.astype(float), out_shape).astype(np.float32)
    s = torch.from_numpy(src).to(DEV)
    lib = L.load()
    ins, outs = _i3(in_shape), _i3(out_shape)
    ws_bytes = lib.mdt_pp_resample_workspace_bytes(ins, outs)
    n_out = int(np.prod(out_shape))

    def call(o, ws):
        return lib.mdt_pp_resample(_DT[dt], L.ptr(s), ins, outs, o[0], ws, ws_bytes, L.stream_ptr())
    got, = _run_guarded(call, [4 * n_out], ws_bytes if ws_bytes else None)
    got = got.view(torch.float32).cpu().numpy().reshape(out_shape)
    u = _ulps(got, want)
    print('resample %s -> %s %s: %d of %d voxels differ, max %.1f ulp' % (in_shape, out_shape, np.dtype(dt), int((u > 0).sum()), u.size, u.max()))
    assert u.max() <= 1


def test_resample_rejects_bad_arguments():
    lib = L.load()
    s = torch.zeros(8, dtype=torch.int16, device=DEV)
    o = torch.zeros(8, dtype=torch.float32, device=DEV)
    two = _i3((2, 2, 2))
    assert lib.mdt_pp_resample(3, L.ptr(s), two, two, L.ptr(o), None, 0, L.stream_ptr()) == -1        # fp64 source
    assert lib.mdt_pp_resample(4, L.ptr(s), _i3((2, 0, 2)), two, L.ptr(o), None, 0, L.stream_ptr()) == -1
    big, tiny = _i3((200, 2, 2)), _i3((1, 2, 2))                                                           # radius 100 > 64
    assert lib.mdt_pp_resample_workspace_bytes(big, tiny) == 0
    assert lib.mdt_pp_resample(4, L.ptr(s), big, tiny, L.ptr(o), None, 0, L.stream_ptr()) == -3
    down = _i3((4, 2, 2))
    assert lib.mdt_pp_resample_workspace_bytes(down, two) == 8 * 16
    assert lib.mdt_pp_resample(4, L.ptr(s), down, two, L.ptr(o), L.ptr(o), 8 * 16 - 1, L.stream_ptr()) == -2


def test_resample_lidc_size():
    """512 x 512 x 300 int16 at (0.55, 0.55, 1.0): a stratified sample, every corner and samples of every face against fp64 point-wise"""
    shape = (300, 512, 512)
    rs = np.random.RandomState(7)
    src = rs.randint(-1100, 1500, shape).astype(np.int16)
    out_shape = P.target_shape(shape, (0.55, 0.55, 1.0), (0.7, 0.7, 1.25))
    assert out_shape == [240, 402, 402]
    got = P.CudaOps(DEV).resample(torch.from_numpy(src).to(DEV), out_shape).cpu().numpy()
    pts = [np.stack([rs.randint(0, s, 20000) for s in out_shape], 1)]
    pts.append(np.array([[a, b, c] for a in (0, out_shape[0] - 1) for b in (0, out_shape[1] - 1) for c in (0, out_shape[2] - 1)]))
    for ax in range(3):
        for end in (0, out_shape[ax] - 1):
            p = np.stack([rs.randint(0, s, 3000) for s in out_shape], 1)
            p[:, ax] = end
            pts.append(p)
    pts = np.concatenate(pts)
    want = PO.resize_points(src, out_shape, pts).astype(np.float32)
    u = _ulps(got[tuple(pts.T)], want)
    print('resample 512x512x300: %d of %d sampled voxels differ, max %.1f ulp' % (int((u > 0).sum()), u.size, u.max()))
    assert u.max() <= 1


# ------------------------------------------------------------------------------------------------------------------- normalisation
def _normalize_guarded(x):
    """every base offset and workspace fill; returns (outputs, stats) of every run"""
    lib = L.load()
    n = x.size
    xb = torch.from_numpy(x.view(np.uint8).copy()).to(DEV)
    ws_bytes = lib.mdt_pp_normalize_workspace_bytes(n)
    runs = []
    for off in OFFSETS:
        for fill in (POISON, 0):
            xg, st, ws = _Guarded(4 * n, off, 0), _Guarded(16, off, POISON), _Guarded(ws_bytes, off, fill)
            xg.data().copy_(xb)
            L.check(lib.mdt_pp_normalize(xg.ptr(), n, st.ptr(), ws.ptr(), ws_bytes, L.stream_ptr()))
            torch.cuda.synchronize()
            for b in (xg, st, ws):
                b.check_guards()
            runs.append((xg.data().cpu().numpy().view(np.float32).copy(), st.data().cpu().numpy().view(np.float64).copy()))
    return runs


@pytest.mark.parametrize('n', [1, 1000, 1025, 262147, 5_000_000])
def test_normalize(n):
    rs = np.random.RandomState(n)
    x = (rs.normal(-400, 700, n) + np.where(rs.rand(n) < 0.02, 3000, 0)).astype(np.float32)
    runs = _normalize_guarded(x)
    y, stats = runs[0]
    for y2, s2 in runs[1:]:
        assert np.array_equal(y.view(np.uint32), y2.view(np.uint32)) and np.array_equal(stats.view(np.uint64), s2.view(np.uint64))
    xc = np.clip(x, -1200, 600).astype(np.float32)
    mean, std = PO.device_stats(xc)
    assert abs(stats[0] - mean) <= 1e-12 * abs(mean) and abs(stats[1] - std) <= 1e-12 * max(std, 1e-300)
    if std == 0:
        return
    want = (xc - np.float32(stats[0])) / np.float32(stats[1]).astype(np.float16)
    u = _ulps(y, want)
    print('normalize n=%d: %d of %d values differ' % (n, int((u > 0).sum()), n))
    assert u.max() <= 1
    ref = (xc - np.mean(xc)) / np.std(xc).astype(np.float16)
    assert np.abs(y - ref).max() <= 2e-6 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------------------------- vote
def _rater_volumes(rs, shape, n):
    """resampled-mask-like fp32 volumes: soft blobs with exact 0.5 / 0.25 steps and continuous values, many sums at 2.0"""
    vols = []
    for _ in range(n):
        v = np.zeros(shape, np.float32)
        c = [rs.randint(0, s) for s in shape]
        z, y, x = np.ogrid[:shape[0], :shape[1], :shape[2]]
        d = ((z - c[0]) / 3.0) ** 2 + ((y - c[1]) / 5.0) ** 2 + ((x - c[2]) / 6.0) ** 2
        v[d <= 1.5] = rs.choice([0.25, 0.5, 0.75, 1.0], size=int((d <= 1.5).sum()))
        v[d <= 0.8] = np.clip(1.2 - d[d <= 0.8], 0, 1).astype(np.float32)
        vols.append(v)
    return vols


@pytest.mark.parametrize('shape,raters', [((9, 21, 35), [2, 1, 5, 4]), ((1, 1, 1), [1]), ((33, 7, 70), [3, 4, 4, 1, 2, 6, 4])])
def test_vote_matches_oracle(shape, raters):
    rs = np.random.RandomState(sum(shape) + len(raters))
    rois = [_rater_volumes(rs, shape, k) for k in raters]
    if shape == (1, 1, 1):
        rois = [[np.full(shape, 0.5, np.float32)] * 4 for _ in range(3)] + [[np.full(shape, 0.499999, np.float32)] * 4]
    st = dict(labels=np.zeros(shape, np.uint8), kept=[])
    boundary = 0
    for vols in rois:
        s = vols[0].copy()
        for v in vols[1:]:
            s += v
        boundary += int((np.abs(s - np.float32(2.0)) <= np.spacing(np.float32(2.0))).sum())
        v = PO.vote(vols)
        kept = bool(v.sum() > 0)
        if kept:
            st['labels'][v >= 0.5] = 1 + sum(st['kept'])
        st['kept'].append(kept)
    want_lab = st['labels']
    n = int(np.prod(shape))
    lib = L.load()
    dev = [[torch.from_numpy(v).to(DEV) for v in vols] for vols in rois]

    def call(o, ws):
        lab, kept, slice_nz, present = o
        for r, vols in enumerate(dev):
            for k, v in enumerate(vols):
                rc = lib.mdt_pp_vote_add(ws, L.ptr(v), n, int(k == 0), L.stream_ptr())
                if rc:
                    return rc
            rc = lib.mdt_pp_vote_label(ws, n, len(vols), r, lab, kept, L.stream_ptr())
            if rc:
                return rc
        return lib.mdt_pp_label_summary(lab, shape[0], n // shape[0], slice_nz, present, L.stream_ptr())
    lab, kept, slice_nz, present = _run_guarded(call, [n, 4 * len(rois), shape[0], 256], 4 * n)
    lab = lab.cpu().numpy().reshape(shape)
    diff = int((lab != want_lab).sum())
    print('vote %s: %d voxels at a rater sum within 1 ulp of 2.0, %d labels differ' % (shape, boundary, diff))
    assert diff == 0
    assert kept.view(torch.int32).cpu().numpy().tolist() == [int(k) for k in st['kept']]
    assert np.array_equal(slice_nz.cpu().numpy() != 0, (want_lab != 0).reshape(shape[0], -1).any(axis=1))
    want_present = np.zeros(256, bool)
    want_present[np.unique(want_lab)] = True
    assert np.array_equal(present.cpu().numpy() != 0, want_present)


def test_vote_rejects_bad_arguments():
    lib = L.load()
    a = torch.zeros(4, dtype=torch.float32, device=DEV)
    lab = torch.zeros(4, dtype=torch.uint8, device=DEV)
    kept = torch.zeros(256, dtype=torch.int32, device=DEV)
    assert lib.mdt_pp_vote_label(L.ptr(a), 4, 0, 0, L.ptr(lab), L.ptr(kept), L.stream_ptr()) == -1
    assert lib.mdt_pp_vote_label(L.ptr(a), 4, 4, 255, L.ptr(lab), L.ptr(kept), L.stream_ptr()) == -3
    assert lib.mdt_pp_vote_add(L.ptr(a), None, 4, 1, L.stream_ptr()) == -1
    assert lib.mdt_pp_label_summary(L.ptr(lab), 0, 4, L.ptr(lab), L.ptr(kept), L.stream_ptr()) == -1


# ------------------------------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return pickle.load(f)


@pytest.fixture(scope='module')
def pp(tmp_path_factory):
    from medicaldetectiontoolkit_b200.configs import make_cf
    root = str(tmp_path_factory.mktemp('lidc'))
    raw = PC.make_raw_dir(root)
    out = []
    for k in range(2):
        cf = make_cf(exp='lidc_exp')
        cf.root_dir, cf.raw_data_dir, cf.pp_dir = root, raw, os.path.join(root, 'pp%d' % k)
        P.preprocess_lidc(cf, read_image=PC.npy_reader)
        out.append(cf.pp_dir)
    return root, raw, out


def test_preprocess_lidc_matches_golden(golden, pp):
    root, raw, (pp_dir, _) = pp
    for pid, want in golden['patients'].items():
        rois = np.load(os.path.join(pp_dir, '%s_rois.npy' % pid))
        img = np.load(os.path.join(pp_dir, '%s_img.npy' % pid))
        assert rois.dtype == np.uint8 and np.array_equal(rois, want['rois']), pid
        # the device image within 1 ulp of the oracle with the device's statistics; the golden's numpy statistics differ from those in the
        # last bit of the fp32 mean at most (tests/test_preprocess_cpu.py), which bounds the difference to the golden
        ct, sp = PC.npy_reader(os.path.join(raw, pid, '%s_ct_scan.nrrd' % pid))
        x = PO.resample_array(ct, sp, PC.TARGET_SPACING)
        want_dev, m_dev, s16 = PO.normalize(x, 'device')
        _, m_np, _ = PO.normalize(x, 'numpy')
        u = _ulps(img, want_dev)
        print('%s: %d of %d image voxels differ from the oracle, max %.1f ulp' % (pid, int((u > 0).sum()), u.size, u.max()))
        assert img.dtype == np.float32 and u.max() <= 1
        # one fp32 rounding of x - mean, the difference of the means, both over the std, and one rounding of the division
        xc = np.clip(x, -1200, 600).astype(np.float32)
        tol = (np.spacing(np.abs(xc - m_np)) + abs(float(m_dev) - float(m_np))) / float(s16) + np.spacing(np.abs(want['img']))
        assert np.all(np.abs(img.astype(np.float64) - want['img']) <= tol), pid
        with open(os.path.join(pp_dir, 'meta_info_%s.pickle' % pid), 'rb') as f:
            meta = pickle.load(f)
        assert meta['pid'] == pid and meta['spacing'] == want['meta']['spacing'] and meta['fg_slices'] == want['meta']['fg_slices']
        assert np.array_equal(meta['class_target'], want['meta']['class_target'])
    with open(os.path.join(pp_dir, 'suppressed_rois.txt')) as f:
        assert f.read() == golden['suppressed']
    import pandas as pd
    df = pd.read_pickle(os.path.join(pp_dir, 'info_df.pickle'))
    assert list(df.pid) == golden['info_df']['pid']


def test_preprocess_lidc_is_reproducible(pp):
    _, _, (a, b) = pp
    names = sorted(f for f in os.listdir(a) if f.endswith('.npy'))
    assert names == sorted(f for f in os.listdir(b) if f.endswith('.npy')) and len(names) == 8
    for f in names:
        with open(os.path.join(a, f), 'rb') as fa, open(os.path.join(b, f), 'rb') as fb:
            assert fa.read() == fb.read(), f


class _Log:
    def info(self, *a, **k):
        pass

    warning = info


def test_preprocessed_directory_feeds_training_and_prediction(pp, tmp_path):
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import predictor, retina_unet
    from medicaldetectiontoolkit_b200.configs import make_cf
    _, _, (pp_dir, _) = pp
    cf = make_cf('retina_unet', 3, (64, 64, 32), exp='lidc_exp')
    cf.pre_crop_size = [72, 72, 40]
    cf.batch_size = 2
    cf.pp_data_path = cf.pp_test_data_path = pp_dir
    cf.exp_dir = cf.fold_dir = str(tmp_path)
    cf.select_prototype_subset = None
    cf.n_cv_splits = 4             # four patients: one test, one validation and two training patients per fold
    cf.batch_sample_slack = 1.0     # free draws: the class balancing redraws forever when no training patient has more benign than malignant ROIs
    gens = D.get_train_generators(cf, _Log())
    torch.manual_seed(0)
    net = retina_unet.net(cf, None).to(DEV)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    res = net.train_forward(next(gens['train']))
    opt.zero_grad()
    res['torch_loss'].backward()
    opt.step()
    assert np.isfinite(res['monitor_values']['loss'])
    for k, v in dict(test_aug=False, merge_2D_to_3D_preds=False, merge_3D_iou=0.1, return_masks_in_test=False, wcs_iou=1e-5, fold=0,
                     test_n_epochs=1, folds=[0]).items():
        setattr(cf, k, v)
    os.makedirs(os.path.join(str(tmp_path), '1_best_checkpoint'))
    torch.save(net.state_dict(), os.path.join(str(tmp_path), '1_best_checkpoint', 'params.pth'))
    np.save(os.path.join(str(tmp_path), 'epoch_ranking.npy'), np.array([1]))
    gen = D.get_test_generator(cf, _Log())
    gen['n_test'] = 1
    got = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(gen)
    assert len(got) == 1
