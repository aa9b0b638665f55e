"""The toy generator on the host: the oracle and the package's generate_experiment (with a numpy stand-in for the device) against the golden
of the reference's own generate_toys.py (tests/golden/make_toys_golden.py), an executable model of csrc/toys.cu's MT19937 against numpy's
RandomState word for word, and the argument checks that run before any launch."""
import gzip
import hashlib
import json
import os
import pickle

import numpy as np
import pandas as pd
import pytest

import _toys_cases as TC
from _toys_cases import TO
from medicaldetectiontoolkit_b200 import generate_toys as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'toys.json.gz')
CASE_NAMES = [c[0] for c in TC.CASES]


@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return json.loads(f.read())


def test_cases_cover_the_regimes(golden):
    assert sorted(golden) == sorted(CASE_NAMES)
    for name, mode, diameters, seed, n in TC.CASES:
        for split in TC.SPLITS:
            assert {im['meta'][1] for im in golden[name][split]['images']} == {0, 1}, (name, split)
    full = lambda r: int(((np.mgrid[-r:r + 1, -r:r + 1] ** 2).sum(0) < r * r).sum())
    sums = lambda name: [(im['meta'][1], im['seg_sum']) for s in TC.SPLITS for im in golden[name][s]['images']]
    assert any(s < full(30) for c, s in sums('shape_5_30') if c == 1)                 # a disc cut by the border
    assert {s for c, s in sums('shape_3_3')} == {0.0, full(3)}                        # class 1's hole clears its whole (smaller) disc
    assert {s for c, s in sums('pattern_0_20') if c == 0} == {0.0}
    assert full(20) - full(4) in {s for c, s in sums('donuts_shape') if c == 1}       # the hole clears the seg ...
    assert full(20) in {s for c, s in sums('donuts_shape_noise') if c == 1}           # ... only in donuts_shape


@pytest.mark.parametrize('name', CASE_NAMES)
def test_oracle_matches_golden(golden, name):
    _, mode, diameters, seed, n = TC.CASES[CASE_NAMES.index(name)]
    for s, split in enumerate(TC.SPLITS):
        for six, want in enumerate(golden[name][split]['images']):
            out, (cx, cy, cls) = TO.image([seed, s, six], mode, diameters)
            assert TO.npy_sha256(out) == want['sha256'], (name, split, six)
            assert cls == want['meta'][1] and float(out[1].sum()) == want['seg_sum']
            assert TO.margin_of(diameters) <= min(cx, cy) and max(cx, cy) < 320 - TO.margin_of(diameters)


def _check_experiment(golden, root, name):
    for split in TC.SPLITS:
        d = os.path.join(root, name, split)
        want = golden[name][split]
        for six, im in enumerate(want['images']):
            path = os.path.join(d, '%d.npy' % six)
            with open(path, 'rb') as f:
                assert hashlib.sha256(f.read()).hexdigest() == im['sha256'], (name, split, six)
            with open(os.path.join(d, 'meta_info_%d.pickle' % six), 'rb') as f:
                meta = pickle.load(f)
            assert [type(v).__name__ for v in meta] == im['meta_types'] == ['str', 'int', 'str']
            assert meta[0] == path and [os.path.relpath(meta[0], root), meta[1], meta[2]] == im['meta']
        df = pd.read_pickle(os.path.join(d, 'info_df.pickle'))
        assert list(df.columns) == want['columns'] == G.META_COLUMNS
        assert [[os.path.relpath(p, root), c, pid] for p, c, pid in zip(df['path'], df['class_id'], df['pid'])] == want['info_df']
        assert list(df['pid']) == sorted(str(i) for i in range(len(want['images'])))


@pytest.mark.parametrize('chunk', [G.CHUNK, 5])
def test_package_with_numpy_ops_matches_golden(golden, tmp_path, monkeypatch, chunk):
    monkeypatch.setattr(G, 'CHUNK', chunk)
    for name, mode, diameters, seed, n in TC.CASES:
        G.generate_experiment(str(tmp_path), name, n, n, mode, class_diameters=diameters, seed=seed, ops=TC.NumpyOps())
        _check_experiment(golden, str(tmp_path), name)


def test_impossible_margin_raises_before_any_launch(tmp_path):
    class NoOps(object):
        def images(self, *a):
            raise AssertionError('launched')
        staging = images
    for diameters in [(320, 320), (0, 321), (20, 1000)]:
        with pytest.raises(ValueError, match='low >= high'):
            G.create_images([[0, 0, 0]], 'donuts_shape', diameters)
        with pytest.raises(ValueError, match='low >= high'):
            G.generate_experiment(str(tmp_path), 'x', 2, 2, 'donuts_shape', diameters, ops=NoOps())
        m = max(diameters) // 2
        with pytest.raises(ValueError):
            np.random.RandomState(0).randint(m, 320 - m)
    assert G.margin_of((318, 0)) == 159 and G.margin_of((19, 20)) == 10
    for bad in [(-2, 20), (20,), (2.5, 20), (2 ** 31, 0)]:
        with pytest.raises((ValueError, TypeError)):
            G.margin_of(bad)
    for keys in [[[0, 0]], [[0, 0, -1]], [[2 ** 32, 0, 0]], [[0.5, 0, 0]], np.zeros((0, 3), int)]:
        with pytest.raises(ValueError):
            G.create_images(keys, 'circles', (20, 20))
    with pytest.raises(ValueError):
        G.generate_experiment(str(tmp_path), 'x', 1, 1, 'circles', seed=-1, ops=NoOps())
    assert not os.listdir(str(tmp_path))


def test_mode_flags():
    assert G.mode_flags('donuts_shape') == G.HOLE | G.HOLE_CLEARS_SEG
    assert G.mode_flags('donuts_pattern') == G.mode_flags('donuts_shape_noise') == G.HOLE
    assert G.mode_flags('circles_scale') == G.mode_flags('circles') == 0


# ---------------------------------------------------------------------------------------------------------- the kernel's MT19937 model
# csrc/toys.cu restated step for step: the serial init_by_array of one thread, the twist as three blocks of words computed from the words
# read before the block's barrier, the 53-bit doubles from word pairs, and thread 0's rejection loop that twists when the state runs out.
N, M = 624, 397


def seed_model(key):
    mt = [0] * N
    prev = mt[0] = 19650218
    for i in range(1, N):
        prev = (1812433253 * (prev ^ (prev >> 30)) + i) & 0xFFFFFFFF
        mt[i] = prev
    i, j, prev = 1, 0, mt[0]
    for _ in range(N):
        prev = ((mt[i] ^ (((prev ^ (prev >> 30)) * 1664525) & 0xFFFFFFFF)) + key[j] + j) & 0xFFFFFFFF
        mt[i] = prev
        i, j = i + 1, j + 1
        if i >= N:
            mt[0], i = mt[N - 1], 1
        if j >= len(key):
            j = 0
    for _ in range(N - 1):
        prev = ((mt[i] ^ (((prev ^ (prev >> 30)) * 1566083941) & 0xFFFFFFFF)) - i) & 0xFFFFFFFF
        mt[i] = prev
        i += 1
        if i >= N:
            mt[0], i = mt[N - 1], 1
    mt[0] = 0x80000000
    return np.array(mt, dtype=np.uint32)


def _term(hi, lo):
    y = (hi & np.uint32(0x80000000)) | (lo & np.uint32(0x7FFFFFFF))
    return (y >> np.uint32(1)) ^ np.where(y & np.uint32(1), np.uint32(0x9908B0DF), np.uint32(0)).astype(np.uint32)


def twist_model(mt):
    old = mt.copy()                                      # every thread's reads before the first barrier
    ta, a_src = _term(old[0:227], old[1:228]), old[397:624]
    tb = _term(old[227:454], old[228:455])
    tc, c_hi = _term(old[454:623], old[455:624]), old[623]
    mt[0:227] = a_src ^ ta                               # block A
    mt[227:454] = mt[0:227] ^ tb                         # block B: word k - 227 is new
    tc = np.append(tc, _term(c_hi, mt[0]))              # word 623 takes the new word 0
    mt[454:624] = mt[227:397] ^ tc                       # block C


def temper(y):
    y = y ^ (y >> np.uint32(11))
    y = y ^ ((y << np.uint32(7)) & np.uint32(0x9D2C5680))
    y = y ^ ((y << np.uint32(15)) & np.uint32(0xEFC60000))
    return y ^ (y >> np.uint32(18))


def pairs_model(mt, n_pairs):
    w = temper(mt[:2 * n_pairs]).astype(np.int64)
    return ((w[0::2] >> 5) * 67108864.0 + (w[1::2] >> 6)) / 9007199254740992.0


def draws_model(mt, pos, margin):
    """thread 0's three draws from word pos on, the CTA twisting whenever the state runs out; returns (cx, cy, class_id), pos after"""
    rng_c = 320 - 2 * margin - 1
    got = []
    while True:
        while len(got) < 3 and pos < N:
            rng, low = (rng_c, margin) if len(got) < 2 else (1, 0)
            if rng == 0:
                got.append(low)
                continue
            mask = rng
            for s in (1, 2, 4, 8, 16):
                mask |= mask >> s
            v = int(temper(mt[pos:pos + 1])[0]) & mask
            pos += 1
            if v <= rng:
                got.append(low + v)
        if len(got) == 3:
            return tuple(got), pos
        twist_model(mt)
        pos = 0


def image_model(key, margin):
    mt = seed_model(key)
    doubles = []
    for _ in range(328):
        twist_model(mt)
        doubles.append(pairs_model(mt, 312))
    twist_model(mt)
    doubles.append(pairs_model(mt, 64))
    params, pos = draws_model(mt, 128, margin)
    return np.concatenate(doubles).reshape(320, 320), params, mt, pos


@pytest.mark.parametrize('key,margin', [([0, 0, 0], 10), ([1, 1, 599], 10), ([2 ** 32 - 1, 7, 123456], 15), ([20261018, 0, 5], 1),
                                        ([3, 1, 0], 0), ([9, 0, 4], 159)])
def test_kernel_model_matches_random_state(key, margin):
    rs = np.random.RandomState(key)
    name, words, pos0 = rs.get_state()[:3]
    assert pos0 == N and np.array_equal(seed_model(key), words)
    img, params, mt, pos = image_model(key, margin)
    want = rs.rand(320, 320)
    assert np.array_equal(img.view(np.uint64), want.view(np.uint64))
    assert params == (rs.randint(margin, 320 - margin), rs.randint(margin, 320 - margin), rs.randint(0, 2))
    _, words, pos_after = rs.get_state()[:3]
    assert pos == pos_after and np.array_equal(mt, words)


@pytest.mark.parametrize('pos', [600, 621, 622, 623, 624])
def test_rejection_loop_model_crosses_into_the_next_twist(pos):
    for key in range(8):
        start = seed_model([key, 1, 2])
        for _ in range(key % 3):
            twist_model(start)
        for margin in (10, 96):                          # ranges 299 and 127: about 41 % and none of the words rejected
            rs = np.random.RandomState()
            rs.set_state(('MT19937', start.copy(), pos))
            want = (rs.randint(margin, 320 - margin), rs.randint(margin, 320 - margin), rs.randint(0, 2))
            mt = start.copy()
            got, pos_after = draws_model(mt, pos, margin)
            assert got == want
            assert (pos_after, list(mt)) == (rs.get_state()[2], list(rs.get_state()[1]))
