"""csrc/loader.cu and data_loader.py on the GPU: the foreground index and the gather bit for bit against numpy through guarded, poisoned
exact-size buffers; BatchGenerator and PatientBatchIterator against the goldens of the reference's loaders; and the generators feeding train
steps and Predictor.predict_test_set end to end."""
import ctypes
import gzip
import json
import os

import numpy as np
import pytest
import torch

import _loader_cases as LC
from _guarded import DEV, _run_guarded
from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import data_loader as D

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'loader.json.gz')


def _np_index(seg):
    return LC.NumpyOps().fg_index(seg)


def _fg_index_guarded(seg):
    Z, Y, X = seg.shape
    want_counts, want_order = _np_index(seg)
    n_fg = len(want_order)
    s = torch.from_numpy(seg).to(DEV)
    lib = L.load()
    ws_bytes = lib.mdt_loader_fg_index_workspace_bytes(Z, Y, X)

    def call(outs, ws):
        return lib.mdt_loader_fg_index(L.ptr(s), Z, Y, X, outs[0], outs[1], n_fg, ws, ws_bytes, L.stream_ptr())
    counts, order = _run_guarded(call, [256 * 4, 4 * n_fg if n_fg else None], ws_bytes, offsets=(0, 256))
    assert np.array_equal(counts.view(torch.int32).cpu().numpy(), want_counts)
    if n_fg:
        assert np.array_equal(order.view(torch.int32).cpu().numpy(), want_order)


@pytest.mark.parametrize('shape,kind', [((7, 5, 3), 'dense'), ((33, 70, 45), 'sparse'), ((20, 31, 97), 'empty'), ((40, 64, 64), 'all255'),
                                        ((3, 2, 1), 'full')])
def test_fg_index_matches_numpy(shape, kind):
    rs = np.random.RandomState(sum(shape))
    if kind == 'empty':
        seg = np.zeros(shape, np.uint8)
    elif kind == 'full':
        seg = rs.randint(1, 256, shape).astype(np.uint8)
    elif kind == 'all255':
        seg = np.where(rs.rand(*shape) < 0.3, rs.randint(1, 256, shape), 0).astype(np.uint8)
    elif kind == 'dense':
        seg = rs.randint(0, 4, shape).astype(np.uint8)
    else:
        seg = np.where(rs.rand(*shape) < 0.02, rs.randint(1, 8, shape), 0).astype(np.uint8)
    _fg_index_guarded(seg)


def test_fg_index_lidc_size():
    """a 512 x 512 x 250 patient with 255 labels, through CudaOps as the loader calls it"""
    rs = np.random.RandomState(3)
    seg = np.zeros((250, 512, 512), np.uint8)
    for k in range(1, 256):
        z, y, x = rs.randint(0, 240), rs.randint(0, 500), rs.randint(0, 500)
        seg[z:z + rs.randint(1, 10), y:y + rs.randint(1, 12), x:x + rs.randint(1, 12)] = k
    counts, order = D.CudaOps(DEV).fg_index(seg)
    want_counts, want_order = _np_index(seg)
    assert np.array_equal(counts, want_counts) and np.array_equal(order, want_order)


def test_fg_index_rejects_bad_arguments():
    lib = L.load()
    s = torch.zeros(8, dtype=torch.uint8, device=DEV)
    c = torch.empty(256, dtype=torch.int32, device=DEV)
    ws = torch.empty(lib.mdt_loader_fg_index_workspace_bytes(2, 2, 2), dtype=torch.uint8, device=DEV)
    null = ctypes.c_void_p(0)
    assert lib.mdt_loader_fg_index(null, 2, 2, 2, L.ptr(c), null, 0, L.ptr(ws), ws.numel(), L.stream_ptr()) == -1
    assert lib.mdt_loader_fg_index(L.ptr(s), 2, 2, 2, L.ptr(c), null, 4, L.ptr(ws), ws.numel(), L.stream_ptr()) == -1
    assert lib.mdt_loader_fg_index(L.ptr(s), 2, 2, 2, L.ptr(c), null, 0, L.ptr(ws), ws.numel() - 1, L.stream_ptr()) == -2
    assert lib.mdt_loader_fg_index(L.ptr(s), 7000, 2, 2, L.ptr(c), null, 0, L.ptr(ws), ws.numel(), L.stream_ptr()) == -3


DT = {0: np.uint8, 1: np.float16, 2: np.float32, 3: np.float64}


def _gather_case(rs, n, C, I, J, K, ext, context=False):
    """random per-element sources and tables that cross every border (-1, past the end), wrap (a last-row entry first) and, with context,
    stack z slices into channels"""
    elems, tabs = [], [[], [], [], []]
    for b in range(n):
        c, z, y, x = ext
        tc = rs.randint(-1, c + 1, C)
        if context:
            s = rs.randint(0, z)
            tz = np.repeat((np.arange(C) - C // 2 + s)[:, None], K, 1)
            tz[(tz < 0) | (tz >= z)] = -1
        else:
            tz = np.tile(np.arange(K) + rs.randint(-3, z - K + 4), (C, 1))
        ty = np.arange(I) + rs.randint(-3, max(1, y - I + 4))
        ty[0] = y - 1                                   # np.take(range(-1, ...)): the window starts at the last row
        tx = np.arange(J) + rs.randint(-5, max(1, x - J + 6))
        for t, v in zip(tabs, (tc, tz, ty, tx)):
            t.append(v.astype(np.int32))
        elems.append(ext)
    return D._src_desc(elems), tuple(np.stack(t) for t in tabs)


@pytest.mark.parametrize('src_dt,out_dt', [(2, 2), (1, 1), (3, 1), (2, 1), (0, 0), (3, 0), (1, 2), (3, 3), (0, 3)])
@pytest.mark.parametrize('geom', [(3, 2, 17, 40, 33, (2, 30, 21, 45), False), (4, 5, 19, 37, 1, (1, 9, 23, 41), True),
                                  (2, 1, 5, 70, 65, (1, 70, 8, 66), False)])
def test_gather_matches_numpy(src_dt, out_dt, geom):
    n, C, I, J, K, ext, context = geom
    rs = np.random.RandomState(n * 7 + src_dt * 3 + out_dt)
    elems, tabs = _gather_case(rs, n, C, I, J, K, ext, context)
    vol = np.abs(rs.randn(n * int(np.prod(ext))) * 40).astype(DT[src_dt]) if src_dt else rs.randint(0, 256, n * int(np.prod(ext))).astype(np.uint8)
    want = LC.NumpyOps().gather(vol, elems, tabs, DT[out_dt])
    src = torch.from_numpy(vol).to(DEV)
    meta = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (elems.view(np.uint8),) + tabs]
    out_bytes = want.nbytes
    lib = L.load()

    def call(outs, ws):
        return lib.mdt_loader_gather(src_dt, L.ptr(src), L.ptr(meta[0]), n, C, I, J, K, L.ptr(meta[1]), L.ptr(meta[2]), L.ptr(meta[3]),
                                     L.ptr(meta[4]), out_dt, outs[0], L.stream_ptr())
    got, = _run_guarded(call, [out_bytes], None, offsets=(0, 256))
    got = got.cpu().numpy().view(DT[out_dt]).reshape(want.shape)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


def test_gather_rejects_bad_arguments():
    lib = L.load()
    t = torch.zeros(64, dtype=torch.int32, device=DEV)
    p = L.ptr(t)
    null = ctypes.c_void_p(0)
    assert lib.mdt_loader_gather(2, p, p, 1, 1, 1, 1, 1, p, p, p, p, 4, p, L.stream_ptr()) == -1
    assert lib.mdt_loader_gather(5, p, p, 1, 1, 1, 1, 1, p, p, p, p, 2, p, L.stream_ptr()) == -1
    assert lib.mdt_loader_gather(2, p, p, 0, 1, 1, 1, 1, p, p, p, p, 2, p, L.stream_ptr()) == -1
    assert lib.mdt_loader_gather(2, p, null, 1, 1, 1, 1, 1, p, p, p, p, 2, p, L.stream_ptr()) == -1
    assert lib.mdt_loader_gather(2, p, p, 1, 1, 70000, 1, 2, p, p, p, p, 2, p, L.stream_ptr()) == -3


# ------------------------------------------------------------------------------------------------------------------- loaders vs goldens
@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return json.loads(f.read())


@pytest.fixture(scope='module')
def dirs(tmp_path_factory):
    root = tmp_path_factory.mktemp('loader')
    out = {}
    for kind in ('lidc', 'pet', 'toy'):
        out[kind] = str(root / kind)
        LC.write_dir(kind, out[kind])
    return out


@pytest.mark.parametrize('name', sorted(LC.CASES))
def test_batch_generator_on_gpu_matches_golden(golden, dirs, name):
    spec = LC.CASES[name]
    cf = LC.case_cf(spec)
    gen = D.BatchGenerator(LC.dataset(spec[0], dirs[spec[0]]), cf.batch_size, cf, seed=0, rank=0, ops=D.CudaOps(DEV))
    for i, want in enumerate(golden['train'][name]):
        b = gen.generate_train_batch()
        assert b['data'].is_cuda and b['seg'].is_cuda
        assert LC.digest(b) == want, (name, i)


@pytest.mark.parametrize('name', sorted(LC.PATIENT_CASES))
def test_patient_batch_iterator_on_gpu_matches_golden(golden, dirs, name):
    spec = LC.PATIENT_CASES[name]
    cf = LC.case_cf(spec)
    it = D.PatientBatchIterator(LC.dataset(spec[0], dirs[spec[0]]), cf, ops=D.CudaOps(DEV))
    for i, want in enumerate(golden['patients'][name]):
        assert LC.digest(it.generate_train_batch()) == want, (name, i)


def test_patient_smaller_than_patch_is_edge_padded(dirs):
    """patients smaller than the patch on some axes: data and seg edge-padded (the numpy stand-in pads by np.pad's rule)"""
    cf = LC.case_cf(('lidc', ('retina_unet', 3, (48, 64, 32), 'lidc_exp'), {}))
    data = LC.dataset('lidc', dirs['lidc'])
    a = D.PatientBatchIterator(data, cf, ops=D.CudaOps(DEV))
    b = D.PatientBatchIterator(data, cf, ops=LC.NumpyOps())
    for pid in list(data):
        x, y = a.generate_train_batch(), b.generate_train_batch()
        assert LC.digest(x) == LC.digest(y), pid
    img = np.load(data['p2']['data']).transpose(1, 2, 0)           # (44, 44, 28) -> (48, 64, 32)
    want = np.pad(img, [(2, 2), (10, 10), (2, 2)], mode='edge')
    it = D.PatientBatchIterator(data, cf, ops=D.CudaOps(DEV))
    it.patient_ix = list(data).index('p2')
    got = it.generate_train_batch()
    assert 'patch_crop_coords' not in got and got['original_img_shape'] == (1, 1, 48, 64, 32)
    assert np.array_equal(got['data'][0, 0], want)


# ------------------------------------------------------------------------------------------------------------------- end to end
class _Log:
    def info(self, *a, **k):
        pass

    warning = info


def _e2e_cf(model, tmp_path, data_dir):
    from medicaldetectiontoolkit_b200.configs import make_cf
    cf = make_cf(model, 3, (64, 64, 32), exp='lidc_exp')
    cf.pre_crop_size = [72, 72, 40]
    cf.batch_size = 2
    cf.pp_data_path = cf.pp_test_data_path = data_dir
    cf.exp_dir = cf.fold_dir = str(tmp_path)
    cf.select_prototype_subset = None
    cf.n_cv_splits = 3
    cf.batch_sample_slack = 1.0     # free draws: the class balancing redraws forever when no training patient has more benign than malignant ROIs
    return cf


@pytest.mark.parametrize('model', ['retina_unet', 'mrcnn'])
def test_train_generators_feed_train_steps(tmp_path, dirs, model):
    from medicaldetectiontoolkit_b200 import mrcnn, retina_unet
    cf = _e2e_cf(model, tmp_path, dirs['lidc'])
    gens = D.get_train_generators(cf, _Log())
    assert set(gens) == {'train', 'val_sampling', 'n_val'} and gens['n_val'] == 50
    torch.manual_seed(0)
    net = (retina_unet if model == 'retina_unet' else mrcnn).net(cf, None).to(DEV)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    for _ in range(2):
        res = net.train_forward(next(gens['train']))
        opt.zero_grad()
        res['torch_loss'].backward()
        opt.step()
        assert np.isfinite(res['monitor_values']['loss'])
    with torch.no_grad():
        res = net.train_forward(next(gens['val_sampling']))
    assert np.isfinite(res['monitor_values']['loss'])


def test_test_generator_feeds_predictor(tmp_path, dirs):
    """two test patients through Predictor.predict_test_set from the GPU loader and from the numpy stand-in's batches: the same boxes"""
    from medicaldetectiontoolkit_b200 import predictor, retina_unet
    cf = _e2e_cf('retina_unet', tmp_path, dirs['lidc'])
    D.get_train_generators(cf, _Log())                      # writes the fold pickle
    for k, v in dict(test_aug=False, merge_2D_to_3D_preds=False, merge_3D_iou=0.1, return_masks_in_test=False, wcs_iou=1e-5, fold=0,
                     test_n_epochs=1, folds=[0]).items():
        setattr(cf, k, v)
    torch.manual_seed(0)
    net = retina_unet.net(cf, None).to(DEV)
    os.makedirs(os.path.join(str(tmp_path), '1_best_checkpoint'))
    torch.save(net.state_dict(), os.path.join(str(tmp_path), '1_best_checkpoint', 'params.pth'))
    np.save(os.path.join(str(tmp_path), 'epoch_ranking.npy'), np.array([1]))
    gen = D.get_test_generator(cf, _Log())
    assert gen['n_test'] >= 2
    gen['n_test'] = 2
    got = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(gen)
    ref_it = D.PatientBatchIterator(gen['test']._data, cf, ops=LC.NumpyOps())
    want = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set({'test': ref_it, 'n_test': 2})
    assert len(got) == len(want) == 2
    assert LC.plain(got) == LC.plain(want)
