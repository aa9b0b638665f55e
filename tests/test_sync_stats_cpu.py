"""Batch statistics across data-parallel ranks without a GPU: parallel.gather_rows and the equal-batch check in gloo worlds of 2 and 3 on CPU
tensors, and an executable numpy model of the per-sample partition of csrc/norm_act.cu (mdt_norm_sample_sums / mdt_norm_stats_from_sums): the
row split of a sample depends on (s, c) only and the sample rows are added in order, so one batch split as 1+1+1+1, 2+2 or 4 gives the same bits."""
import os
import socket
import sys
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(rank, n, k):
    rs = np.random.RandomState(100 + rank)
    r = rs.randn(n, k) * 10.0 ** rs.randint(-300, 300, size=(n, k))
    r[0, 0] = -0.0            # signed zeros and specials keep their bits too
    r[-1, -1] = np.inf
    return torch.from_numpy(r)


def _worker(rank, world, port, q):
    try:
        sys.path.insert(0, ROOT)
        import torch.distributed as dist
        from medicaldetectiontoolkit_b200 import parallel as P
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group('gloo', rank=rank, world_size=world)
        got = P.gather_rows(_rows(rank, 3, 5))
        P.check_equal_batches((2, 1, 64, 64, 32), 'cpu')
        try:
            P.check_equal_batches((1 + (rank == world - 1), 1, 64, 64, 32), 'cpu')
            raised = None
        except RuntimeError as e:
            raised = str(e)
        dist.destroy_process_group()
        q.put((rank, {'rows': got.numpy().copy(), 'raised': raised}))
    except BaseException:
        q.put((rank, traceback.format_exc()))


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_gather_rows_and_equal_batch_check(world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=300) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    want = torch.cat([_rows(r, 3, 5) for r in range(world)])
    for r in range(world):
        assert isinstance(got[r], dict), got[r]
        rows = got[r]['rows']
        assert rows.shape == (3 * world, 5) and rows.dtype == np.float64
        assert np.array_equal(rows.view(np.uint64), want.numpy().view(np.uint64)), r   # rank-major, bit for bit
        assert got[r]['raised'] is not None and 'same input shape' in got[r]['raised'], r    # on every rank


def test_gather_rows_rejects_other_dtypes():
    from medicaldetectiontoolkit_b200 import parallel as P
    with pytest.raises(ValueError):
        P.gather_rows(torch.zeros(2, 3, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------ the partition model
THREADS, TARGET_BLOCKS, MIN_BLOCK_ELEMS, SAMPLE_CHUNKS = 256, 1024, 4096, 512


def _sample_geo(s, c):
    """make_sample_geo: (rows per chunk, chunks) of one sample, from (s, c) alone"""
    min_rows = max(MIN_BLOCK_ELEMS // c, 1)
    chunks = min(-(-s // min_rows), SAMPLE_CHUNKS)
    rows = -(-s // chunks)
    return rows, -(-s // rows)


def _block_partial(v, r0, r1, c):
    """partials_kernel: thread (tr, tc) adds rows r0 + tr, r0 + tr + RP, ... in order; thread rows 1.. are then folded into row 0 in order"""
    ct = min(c, THREADS)
    rp = THREADS // ct
    out = np.zeros(c)
    for c0 in range(0, c, ct):
        cols = v[r0:r1, c0:c0 + ct]
        acc = np.zeros((rp, cols.shape[1]))
        for j in range(0, r1 - r0, rp):
            blk = cols[j:j + rp]
            acc[:blk.shape[0]] += blk          # a thread without a row adds nothing
        tot = acc[0].copy()
        for t in range(1, rp):
            tot += acc[t]
        out[c0:c0 + ct] = tot
    return out


def _group_total(parts):
    """group_total: lane l adds chunks l, l + 32, ... in order, then the xor butterfly 16, 8, 4, 2, 1"""
    lanes = np.zeros((32,) + parts.shape[1:])
    for k in range(parts.shape[0]):
        lanes[k % 32] += parts[k]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return lanes[0]


def _sample_sums(x):
    """mdt_norm_sample_sums of a local batch x [n, s, c] -> [n, c, 2]; nothing below depends on n"""
    n, s, c = x.shape
    rows, chunks = _sample_geo(s, c)
    out = np.zeros((n, c, 2))
    for b in range(n):
        for q, v in enumerate((x[b], x[b] * x[b])):
            parts = np.stack([_block_partial(v, k * rows, min((k + 1) * rows, s), c) for k in range(chunks)])
            out[b, :, q] = _group_total(parts)
    return out


def _stats_from_sums(rows, s):
    """mdt_norm_stats_from_sums: the sample rows added in index order, then mean and biased variance over M = N * s"""
    tot = np.zeros(rows.shape[1:])
    for r in rows:
        tot = tot + r
    m = rows.shape[0] * s
    mu = tot[:, 0] / m
    return mu, np.maximum(tot[:, 1] / m - mu * mu, 0.0)


def _old_batch_sums(x):
    """the unsynchronised partition (make_geo, per_sample = 0): blocks over the n * s rows of the local batch, their count from kTargetBlocks"""
    n, s, c = x.shape
    r = n * s
    min_rows = max(MIN_BLOCK_ELEMS // c, 1)
    chunks = max(min(TARGET_BLOCKS, -(-r // min_rows)), 1)
    rows = -(-r // chunks)
    v = x.reshape(r, c)
    parts = np.stack([_block_partial(v, k * rows, min((k + 1) * rows, r), c) for k in range(-(-r // rows))])
    return _group_total(parts)


@pytest.mark.parametrize("s,c", [(5000, 3), (1200, 18), (64, 576), (30000, 1)])
def test_partition_model_gives_the_same_bits_for_any_split(s, c):
    rs = np.random.RandomState(s + c)
    x = (rs.randn(4, s, c) * 10.0 ** rs.randint(-4, 4, size=(4, s, c)) + 1e3).astype(np.float32).astype(np.float64)   # sums that round
    stats = []
    for split in ((1, 1, 1, 1), (2, 2), (4,)):
        starts = np.cumsum((0,) + split)[:-1]
        gathered = np.concatenate([_sample_sums(x[a:a + k]) for a, k in zip(starts, split)])   # each rank's rows, rank-major
        stats.append(_stats_from_sums(gathered, s))
    for mu, var in stats[1:]:
        assert np.array_equal(mu, stats[0][0]) and np.array_equal(var, stats[0][1])
    ref = x.reshape(-1, c)
    assert np.allclose(stats[0][0], ref.mean(0), rtol=1e-12) and np.allclose(stats[0][1], ref.var(0), rtol=1e-6)


def test_sample_geometry_is_wide_and_batch_free():
    # a sample of the lidc 3D shape at the full-resolution widths gets hundreds of blocks: a per-rank batch of one still fills 132 SMs
    for c in (18, 36, 72):
        rows, chunks = _sample_geo(128 * 128 * 64, c)
        assert chunks == SAMPLE_CHUNKS and rows * chunks >= 128 * 128 * 64
    rows, chunks = _sample_geo(7, 3)
    assert (rows, chunks) == (7, 1)


def test_unsynchronised_partition_depends_on_the_batch():
    """why the per-sample partition exists: the local-batch partition groups rows differently for 2 and 4 samples"""
    rs = np.random.RandomState(1)
    x = (rs.randn(4, 20000, 3) * 10.0 ** rs.randint(-4, 4, size=(4, 20000, 3))).astype(np.float32).astype(np.float64)
    four = _old_batch_sums(x)
    two = _old_batch_sums(x[:2]) + _old_batch_sums(x[2:])
    assert not np.array_equal(four, two)
