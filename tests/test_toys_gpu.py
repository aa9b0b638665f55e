"""csrc/toys.cu and generate_toys.py on the GPU: the C entry point through guarded, poisoned exact-size buffers against oracle/toys_oracle.py
(bit for bit, past one wave of CTAs), every golden case of the reference's own generate_toys.py through create_images, discs cut by the
border and holes outside their disc, launches that split the same keys differently, generate_experiment's files, and a generated experiment
feeding the toy loader, a train step, Predictor.predict_test_set and the Evaluator."""
import gzip
import json
import os
import pickle
import sys

import numpy as np
import pandas as pd
import pytest
import torch

import _toys_cases as TC
from _guarded import DEV, _run_guarded
from _toys_cases import TO
from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import generate_toys as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'toys.json.gz')
IMG_BYTES = 2 * 320 * 320 * 8


def _oracle(keys, mode, diameters, margin):
    outs = [TO.image([int(k) for k in key], mode, diameters, margin) for key in keys]
    return np.stack([o[0] for o in outs]), np.array([o[1] for o in outs], dtype=np.int32).reshape(-1, 3)


def _abi(keys, mode, diameters, margin, offsets=None):
    """mdt_toy_images on keys through guarded buffers: host (img float64 [n, 2, 320, 320], params int32 [n, 3])"""
    n = len(keys)
    k = torch.from_numpy(np.ascontiguousarray(keys, dtype=np.uint32).view(np.int32)).to(DEV)
    lib = L.load()

    def call(o, ws):
        return lib.mdt_toy_images(L.ptr(k), n, margin, int(diameters[0]), int(diameters[1]), G.mode_flags(mode), o[0], o[1], L.stream_ptr())
    kw = {} if offsets is None else {'offsets': offsets}
    img, params = _run_guarded(call, [n * IMG_BYTES, 12 * n], None, **kw)
    return img.cpu().numpy().view(np.float64).reshape(n, 2, 320, 320), params.cpu().numpy().view(np.int32).reshape(n, 3)


def _assert_same(got, want, what):
    gi, gp = got
    wi, wp = want
    assert np.array_equal(gp, wp), what
    bad = np.flatnonzero((gi.view(np.uint64) != wi.view(np.uint64)).reshape(len(gi), -1).any(1))
    assert bad.size == 0, (what, 'images differ:', bad[:10].tolist())


@pytest.mark.parametrize('n', [1, 3, 1200])
def test_abi_matches_oracle(n):
    """1200 images: more than the 1056 CTAs of 256 threads an H100 holds at once"""
    keys = TC.keys(20261018, n % 2, n, start=7)
    mode, diameters = ('donuts_shape', (20, 20)) if n != 3 else ('donuts_pattern', (19, 20))
    got = _abi(keys, mode, diameters, TO.margin_of(diameters), offsets=(256,) if n > 100 else None)
    _assert_same(got, _oracle(keys, mode, diameters, TO.margin_of(diameters)), n)
    if n > 100:
        assert set(got[1][:, 2]) == {0, 1}


def test_abi_rejects_bad_arguments():
    lib = L.load()
    k = torch.zeros(3, dtype=torch.int32, device=DEV)
    img = torch.empty(2 * 320 * 320, dtype=torch.float64, device=DEV)
    p = torch.empty(3, dtype=torch.int32, device=DEV)
    args = lambda **kw: [kw.get(a, d) for a, d in (('keys', L.ptr(k)), ('n', 1), ('margin', 10), ('r0', 20), ('r1', 20), ('flags', 3),
                                                    ('img', L.ptr(img)), ('params', L.ptr(p)))] + [L.stream_ptr()]
    assert lib.mdt_toy_images(*args()) == 0
    for bad in [dict(keys=None), dict(img=None), dict(params=None), dict(n=0), dict(margin=-1), dict(margin=160), dict(r0=-1), dict(r1=-1),
                dict(flags=4)]:
        assert lib.mdt_toy_images(*args(**bad)) == -1, bad
    assert lib.mdt_toy_images(*args(margin=159)) == 0
    torch.cuda.synchronize()


@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return json.loads(f.read())


@pytest.mark.parametrize('name', [c[0] for c in TC.CASES])
def test_create_images_matches_golden(golden, name):
    _, mode, diameters, seed, n = [c for c in TC.CASES if c[0] == name][0]
    for s, split in enumerate(TC.SPLITS):
        img, params = G.create_images(TC.keys(seed, s, n), mode, diameters)
        assert img.is_cuda and img.dtype == torch.float64 and tuple(img.shape) == (n, 2, 320, 320)
        img, params = img.cpu().numpy(), params.cpu().numpy()
        for six, want in enumerate(golden[name][split]['images']):
            assert TO.npy_sha256(img[six]) == want['sha256'], (name, split, six)
            assert int(params[six, 2]) == want['meta'][1] and float(img[six, 1].sum()) == want['seg_sum']


@pytest.mark.parametrize('mode,diameters,margin', [('donuts_shape', (20, 20), 10), ('donuts_pattern', (30, 30), 15), ('circles', (0, 0), 0),
                                                   ('donuts_shape', (3, 2), 0), ('donuts_shape_noise', (1, 3), 1), ('donuts_shape', (5, 9), 159),
                                                   ('circles_scale', (400, 2), 2)])
def test_border_cuts_and_holes_outside_the_disc(mode, diameters, margin):
    keys = TC.keys(77, 1, 300)
    want = _oracle(keys, mode, diameters, margin)
    _assert_same(_abi(keys, mode, diameters, margin, offsets=(0,)), want, (mode, diameters, margin))
    cx, cy, cls = want[1].T
    r = np.where(cls == 1, diameters[1], diameters[0])
    cut = (np.minimum(cx, cy) - r < 0) | (np.maximum(cx, cy) + r > 320)
    if max(diameters) > 0:
        assert cut.any() or margin >= max(diameters), 'no disc reaches the border'
    if 'donuts' in mode and diameters[1] < 4:
        assert (cls == 1).any()                                    # a hole wider than its disc
    if margin == 0:
        assert (np.minimum(cx, cy) == 0).any() or (np.maximum(cx, cy) == 319).any()


def test_launches_do_not_change_the_images():
    keys = TC.keys(3, 0, 600)
    one = G.create_images(keys, 'donuts_shape')
    a = G.create_images(keys[:257], 'donuts_shape')
    b = G.create_images(keys[257:], 'donuts_shape')
    again = G.create_images(keys, 'donuts_shape')
    bits = lambda x: x.view(torch.int64) if x.dtype == torch.float64 else x
    for t in (0, 1):
        assert torch.equal(bits(one[t]), bits(torch.cat([a[t], b[t]]))) and torch.equal(bits(one[t]), bits(again[t]))


def _read(path):
    with open(path, 'rb') as f:
        return f.read()


def test_generate_experiment_writes_the_reference_formats(tmp_path):
    n_train, n_test, seed = 150, 140, 11            # three launches of G.CHUNK images, one with images of both splits
    runs = [str(tmp_path / 'a'), str(tmp_path / 'b')]
    for root in runs:
        G.generate_experiment(root, 'donuts_shape', n_train, n_test, 'donuts_shape', seed=seed)
    for s, (split, n) in enumerate([('train', n_train), ('test', n_test)]):
        d = os.path.join(runs[0], 'donuts_shape', split)
        imgs, params = _oracle(TC.keys(seed, s, n), 'donuts_shape', (20, 20), 10)
        for six in range(n):
            path = os.path.join(d, '%d.npy' % six)
            data = _read(path)
            assert data == TO.npy_bytes(imgs[six]), (split, six)
            assert data == _read(os.path.join(runs[1], 'donuts_shape', split, '%d.npy' % six))
            with open(os.path.join(d, 'meta_info_%d.pickle' % six), 'rb') as f:
                meta = pickle.load(f)
            assert meta == [path, int(params[six, 2]), str(six)] and type(meta[1]) is int
        df = pd.read_pickle(os.path.join(d, 'info_df.pickle'))
        assert list(df.columns) == ['path', 'class_id', 'pid']
        assert list(df['pid']) == sorted(str(i) for i in range(n)) and len(df) == n
        assert list(df['class_id']) == [int(params[int(p), 2]) for p in df['pid']]
        assert sorted(os.listdir(d)) == sorted(os.listdir(os.path.join(runs[1], 'donuts_shape', split)))


# ------------------------------------------------------------------------------------------------------------------- end to end
class _Log:
    def info(self, *a, **k):
        pass

    warning = info


@pytest.fixture(scope='module')
def toy_exp(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('toys'))
    G.generate_experiment(root, 'donuts_shape', 24, 4, 'donuts_shape', seed=5)
    return os.path.join(root, 'donuts_shape')


def _cf(model, exp_dir, tmp_path):
    from medicaldetectiontoolkit_b200.configs import make_cf
    cf = make_cf(model, 2, (320, 320), exp='toy_exp', batch_size=4)
    cf.pp_data_path = os.path.join(exp_dir, 'train')
    cf.pp_test_data_path = os.path.join(exp_dir, 'test')
    cf.exp_dir = cf.fold_dir = str(tmp_path)
    cf.n_train_val_data = 24
    return cf


@pytest.mark.parametrize('model', ['retina_unet', 'mrcnn'])
def test_generated_experiment_feeds_the_toy_loader_and_a_train_step(toy_exp, tmp_path, model):
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import mrcnn, retina_unet
    cf = _cf(model, toy_exp, tmp_path)
    gens = D.get_train_generators(cf, _Log())
    torch.manual_seed(0)
    net = (retina_unet if model == 'retina_unet' else mrcnn).net(cf, None).to(DEV)
    res = net.train_forward(next(gens['train']))
    res['torch_loss'].backward()
    assert np.isfinite(res['monitor_values']['loss'])
    assert all(bool(torch.isfinite(p.grad).all()) for p in net.parameters() if p.grad is not None)
    assert gens['n_val'] == 8
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
    import augment_oracle as AO
    for _ in range(gens['n_val']):
        batch = next(gens['val_patient'])
        out = np.load(os.path.join(cf.pp_data_path, '%s.npy' % batch['pid']))
        with open(os.path.join(cf.pp_data_path, 'meta_info_%s.pickle' % batch['pid']), 'rb') as f:
            class_id = pickle.load(f)[1]
        want = AO.seg_to_boxes(out[1].astype(np.uint8)[None, None], [[class_id]], 2, False, with_masks=False)
        assert len(batch['bb_target'][0]) == 1 and np.array_equal(np.asarray(batch['bb_target'][0]), want['bb_target'][0]), batch['pid']
        assert list(batch['roi_labels'][0]) == [class_id + 1]
        assert np.array_equal(batch['data'][0, 0], out[0])


def test_generated_experiment_feeds_prediction_and_evaluation(toy_exp, tmp_path):
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import evaluator, predictor, retina_unet
    cf = _cf('retina_unet', toy_exp, tmp_path)
    for k, v in dict(test_aug=False, return_masks_in_test=False, wcs_iou=1e-5, fold=0, test_n_epochs=1, folds=[0]).items():
        setattr(cf, k, v)
    torch.manual_seed(0)
    net = retina_unet.net(cf, None).to(DEV)
    os.makedirs(os.path.join(str(tmp_path), '1_best_checkpoint'))
    torch.save(net.state_dict(), os.path.join(str(tmp_path), '1_best_checkpoint', 'params.pth'))
    np.save(os.path.join(str(tmp_path), 'epoch_ranking.npy'), np.array([1]))
    gen = D.get_test_generator(cf, _Log())
    assert gen['n_test'] == 4
    results = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(gen)
    assert sorted(pid for _, pid in results) == ['0', '1', '2', '3']
    ev = evaluator.Evaluator(cf, _Log(), mode='test')
    ev.evaluate_predictions(results)
    stats, _ = ev.return_metrics()
    assert stats[-1]['name'] == 'average_foreground_roi'
    assert set(ev.columns['pid']) == {'0', '1', '2', '3'}        # every patient has a ground-truth box, found or missed
