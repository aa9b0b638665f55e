"""A host restatement of how csrc/norm_act.cu splits a normalisation over blocks and threads, and checks that the split visits every element once.

make_geo / make_sample_geo restate the kernels' functions of the same names: a sample group of R rows is cut into `chunks` blocks of `rows` rows
(the last one may be shorter).  Walk restates the struct of the same name: thread (tr, tc) of a block adds rows r0 + tr, r0 + tr + RP, ... of
channels tc, tc + CT, ... .  group_lanes restates group_total: lane l of the finalising warp folds chunks l, l + 32, ... .
tests/test_norm_edges_gpu.py imports this restatement to assert which regimes of the split its cases reach."""
import itertools
import random
from collections import namedtuple

import numpy as np
import pytest

THREADS = 256
TARGET_BLOCKS = 1024
MIN_BLOCK_ELEMS = 4096
SAMPLE_CHUNKS = 512
WARP = 32

Geo = namedtuple("Geo", "B C R rows chunks")


def _cdiv(a, b):
    return -(-a // b)


def make_geo(n, s, c, per_sample):
    """the block split of mdt_norm_stats / _apply / _backward (and of _backward_from_sums with per_sample = 0); None where the kernel refuses"""
    if n < 1 or s < 1 or c < 1 or n * s > (1 << 40) // c:
        return None
    B = n if per_sample else 1
    R = s if per_sample else n * s
    min_rows = max(MIN_BLOCK_ELEMS // c, 1)
    chunks = max(min(_cdiv(TARGET_BLOCKS, B), _cdiv(R, min_rows)), 1)
    rows = _cdiv(R, chunks)
    g = Geo(B, c, R, rows, _cdiv(R, rows))
    return g if g.B * g.chunks < (1 << 31) else None


def make_sample_geo(n, s, c):
    """the per-sample split of mdt_norm_sample_sums / _backward_sample_sums: a function of (s, c) alone, so a sample's sums do not depend on
    the batch it sits in"""
    if n < 1 or s < 1 or c < 1 or n * s > (1 << 40) // c:
        return None
    min_rows = max(MIN_BLOCK_ELEMS // c, 1)
    chunks = min(_cdiv(s, min_rows), SAMPLE_CHUNKS)
    rows = _cdiv(s, chunks)
    g = Geo(n, c, s, rows, _cdiv(s, rows))
    return g if g.B * g.chunks < (1 << 31) else None


def lanes(c):
    """(CT, RP): channel lanes and row lanes of a block of THREADS threads"""
    ct = min(c, THREADS)
    return ct, THREADS // ct


def last_chunk_rows(g):
    return g.R - (g.chunks - 1) * g.rows


def regimes(g, sample=False):
    """the split regimes a geometry reaches (names used by the coverage assertions of the GPU edge tests)"""
    ct, rp = lanes(g.C)
    out = set()
    if sample:
        wanted = _cdiv(g.R, max(MIN_BLOCK_ELEMS // g.C, 1))
        out |= {"sample-chunks-%d" % g.chunks} if g.chunks in (1, 511, 512) else set()
        if wanted > SAMPLE_CHUNKS:
            out.add("sample-cap")
        return out
    if g.chunks in (1, 32, 33):
        out.add("chunks-%d" % g.chunks)
    elif 2 <= g.chunks <= 31:
        out.add("chunks-2-31")
    if g.B == 1 and g.chunks == TARGET_BLOCKS:
        out.add("bn-cap")
    if g.B == 3 and g.chunks == _cdiv(TARGET_BLOCKS, 3):
        out.add("in3-cap")
    if last_chunk_rows(g) < g.rows:
        out.add("short-last-chunk")
    if g.rows < rp:
        out.add("rows<RP")
    out.add("C=%d" % g.C)
    return out


def walk(g, block, thread):
    """(b, k, CT, RP, tc, tr, r0, r1) of struct Walk for one thread of one block"""
    b, k = block // g.chunks, block % g.chunks
    ct, rp = lanes(g.C)
    r0 = b * g.R + k * g.rows
    return b, k, ct, rp, thread % ct, thread // ct, r0, min(r0 + g.rows, (b + 1) * g.R)


def visit_counts(g):
    """(rows, channels): how often the walk of every block and thread visits each of the B * R rows, and each channel within a row"""
    ct, rp = lanes(g.C)
    row_count = np.zeros(g.B * g.R, dtype=np.int64)
    chan_count = np.zeros(g.C, dtype=np.int64)
    for thread in range(THREADS):   # the channels a thread covers (the same in every block): passes c0 = 0, CT, 2 CT, ...
        _, _, _, _, tc, tr, _, _ = walk(g, 0, thread)
        if tr < rp:
            for c0 in range(0, g.C, ct):
                if c0 + tc < g.C and tr == 0:
                    chan_count[c0 + tc] += 1
    lane_rows = np.arange(rp)[:, None]
    for block in range(g.B * g.chunks):
        _, _, _, _, _, _, r0, r1 = walk(g, block, 0)
        steps = np.arange(_cdiv(max(r1 - r0, 0), rp) + 1)[None, :]
        r = r0 + lane_rows + rp * steps     # row lane tr walks r0 + tr, r0 + tr + RP, ... while r < r1
        np.add.at(row_count, r[r < r1], 1)
    return row_count, chan_count


def group_lanes(g):
    """the chunk indices each lane of the finalising warp folds (group_total): lane l takes l, l + 32, ... < chunks"""
    return [list(range(lane, g.chunks, WARP)) for lane in range(WARP)]


def finalize_warps(g):
    """warps launched by finalize_grid: ceil(B * C * 32 / THREADS) blocks of THREADS threads, one warp per group"""
    return _cdiv(g.B * g.C * WARP, THREADS) * THREADS // WARP


# (n, s, c, per_sample) of tests/test_norm_edges_gpu.py's split matrix, and (n_total, s, c) of its synchronised-path cases
SPLIT_CASES = [
    (2, 100, 3, 0),          # batch norm, 1 chunk; rows 200 >= RP 85
    (2, 20, 3, 0),           # 1 chunk of 40 rows < RP 85
    (3, 4, 18, 1),           # instance norm, 1 chunk of 4 rows < RP 14
    (1, 50, 1, 1),           # C = 1: one channel lane, 256 row lanes, 50 rows
    (3, 777, 27, 0),         # 16 chunks of 146 rows, the last 141
    (2, 256, 256, 0),        # 32 chunks of 16 rows, C = 256
    (3, 176, 256, 0),        # 33 chunks of 16 rows
    (4, 2048, 576, 0),       # the 1024-chunk cap of batch norm: 8 rows per chunk, three channel passes (256, 256, 64)
    (3, 77634, 18, 1),       # instance norm with n = 3: ceil(1024 / 3) = 342 chunks of 227 rows
    (2, 3001, 255, 1),       # C = 255: one idle thread per block; 188 chunks, the last one short
    (5, 333, 257, 0),        # C = 257: a second channel pass of one lane
    (2, 1200, 513, 1),       # C = 513: three passes, the last of one lane
    (1, 40000, 1, 0),        # C = 1 batch norm: 10 chunks of 4000 rows
    (7, 130, 576, 1),        # instance norm, 19 chunks of 7 rows (RP = 1)
]
SYNC_CASES = [               # (n_total, s, c) over which (local_first_row, n) shards are taken
    (4, 300, 18),            # 2 chunks per sample
    (3, 16 * 511, 256),      # 511 chunks per sample
    (2, 16 * 512, 256),      # 512 chunks per sample
    (2, 9000, 256),          # the 512-chunk cap: 563 chunks of 16 rows wanted, 500 of 18 rows taken, the last one short
    (5, 7, 3),               # 1 chunk per sample
    (3, 900, 257),           # C = 257
]

SPLIT_REGIMES = {"chunks-1", "chunks-2-31", "chunks-32", "chunks-33", "bn-cap", "in3-cap", "short-last-chunk", "rows<RP",
                 "C=1", "C=3", "C=255", "C=256", "C=257", "C=513", "C=576"}
SAMPLE_REGIMES = {"sample-chunks-1", "sample-chunks-511", "sample-chunks-512", "sample-cap"}


def covered():
    """(regimes of the split matrix, regimes of the per-sample split) reached by SPLIT_CASES and SYNC_CASES"""
    split = set().union(*(regimes(make_geo(*case)) for case in SPLIT_CASES))
    sample = set().union(*(regimes(make_sample_geo(n, s, c), sample=True) for n, s, c in SYNC_CASES))
    return split, sample


def _random_shapes(count, seed):
    rng = random.Random(seed)
    for _ in range(count):
        c = rng.choice([1, 2, 3, 17, 18, 36, 127, 128, 129, 255, 256, 257, 511, 513, 576, 1000])
        n = rng.randint(1, 9)
        s = rng.choice([1, 2, 3, rng.randint(1, 300), rng.randint(1, 5000), rng.randint(1, 60000) // max(1, c // 16)])
        yield n, max(s, 1), c


def _check_walk(g):
    rows, chans = visit_counts(g)
    assert (rows == 1).all(), ("rows visited", g, int(rows.min()), int(rows.max()))
    assert (chans == 1).all(), ("channels visited", g)
    folded = sorted(itertools.chain.from_iterable(group_lanes(g)))
    assert folded == list(range(g.chunks)), g
    assert finalize_warps(g) >= g.B * g.C
    assert 1 <= g.chunks and (g.chunks - 1) * g.rows < g.R <= g.chunks * g.rows


def test_the_case_lists_reach_every_regime():
    split, sample = covered()
    assert SPLIT_REGIMES <= split, SPLIT_REGIMES - split
    assert SAMPLE_REGIMES <= sample, SAMPLE_REGIMES - sample


@pytest.mark.parametrize("case", SPLIT_CASES, ids=lambda c: "n%d-s%d-c%d-ps%d" % c)
def test_split_cases_visit_every_element_once(case):
    _check_walk(make_geo(*case))


@pytest.mark.parametrize("case", SYNC_CASES, ids=lambda c: "n%d-s%d-c%d" % c)
def test_sample_split_cases_visit_every_element_once(case):
    _check_walk(make_sample_geo(*case))
    _check_walk(make_geo(case[0], case[1], case[2], 0))     # mdt_norm_backward_from_sums walks the batch-norm split


def test_random_shapes_visit_every_element_once():
    for n, s, c in _random_shapes(150, seed=7):
        for per_sample in (0, 1):
            _check_walk(make_geo(n, s, c, per_sample))
        _check_walk(make_sample_geo(n, s, c))


def test_sample_split_does_not_depend_on_the_batch():
    for n, s, c in list(_random_shapes(200, seed=8)) + [(n, s, c) for n, s, c in SYNC_CASES]:
        one = make_sample_geo(1, s, c)
        for m in (2, 3, n, 64):
            g = make_sample_geo(m, s, c)
            assert (g.R, g.rows, g.chunks) == (one.R, one.rows, one.chunks)


def test_the_split_caps():
    """no shape gives more than 1024 chunks for a batch norm, ceil(1024 / n) per instance-norm sample, or 512 per sample of the per-sample
    split"""
    for n, s, c in _random_shapes(300, seed=9):
        bn, inn, smp = make_geo(n, s, c, 0), make_geo(n, s, c, 1), make_sample_geo(n, s, c)
        assert bn.chunks <= TARGET_BLOCKS and inn.chunks <= _cdiv(TARGET_BLOCKS, n) and smp.chunks <= SAMPLE_CHUNKS


def test_refusals():
    assert make_geo(0, 4, 4, 0) is None and make_geo(2, 0, 4, 1) is None and make_geo(2, 4, 0, 0) is None
    assert make_geo(1, 1 << 31, 1 << 10, 0) is None     # more than 2^40 elements
    assert make_sample_geo(0, 4, 4) is None
