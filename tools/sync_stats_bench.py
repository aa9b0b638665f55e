"""Step time of a batch-norm Retina U-Net (lidc 3D shape: per-GPU batch 2 of 128 x 128 x 64) with and without synchronised batch statistics
(parallel.sync_batch_statistics), at world 1 and at the number of GPUs visible, plus the exchanges one synchronised step issues and their bytes.

    python tools/sync_stats_bench.py [--steps 10] [--warmup 3] [--world N] [--out result.json]

One process per GPU (NCCL when every rank has its own GPU; gloo at world 1).  Each step is train_forward + backward + the flat gradient
all-reduce + Adam, timed with a host clock around work that ends in a device synchronise.  Prints one JSON line.

At world 1 a synchronised step issues no collective; its statistics exchanges are still counted (the same calls at any world size, world x
the bytes).  At world >= 2 a step adds one shape check per forward and the gradient all-reduce to them."""
import argparse
import json
import os
import socket
import sys
import time
import traceback

import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _run(rank, world, sync, steps, warmup):
    import torch.distributed as dist
    from medicaldetectiontoolkit_b200 import parallel, retina_unet
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    cf = make_cf('retina_unet', 3, (128, 128, 64))
    cf.norm = 'batch_norm'
    torch.manual_seed(0)
    net = retina_unet.net(cf, None).cuda()
    if sync:
        parallel.sync_batch_statistics(net)
    red = parallel.FlatGradAllReduce(net, world)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    batches = [synthetic_batch(cf, 2, seed=100 * rank + i) for i in range(4)]
    # statistics exchanges: every parallel.all_reduce_rows call (batch norm forward / backward, seg loss forward / backward).  A group of one
    # rank skips the collective itself, but the calls and their buffers are those of any world size, with world x the bytes.
    exch = {'calls': 0, 'bytes': 0}
    real = parallel.all_reduce_rows

    def counting(buf, *a, **k):
        exch['calls'] += 1
        exch['bytes'] += buf.numel() * buf.element_size()
        return real(buf, *a, **k)
    times = []
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        dist.barrier()
        if i == warmup:
            parallel.all_reduce_rows = counting   # count the first timed step's exchanges
        t0 = time.perf_counter()
        red.zero_grad()
        res = net.train_forward(batches[i % len(batches)])
        res['torch_loss'].backward()
        red.all_reduce()
        opt.step()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        if i == warmup:
            parallel.all_reduce_rows = real
            first = dict(exch)
    t = sorted(times[warmup:])
    return {'median_ms': 1e3 * t[len(t) // 2], 'min_ms': 1e3 * t[0], 'max_ms': 1e3 * t[-1], 'stat_exchanges_per_step': first['calls'],
            'stat_exchange_bytes_per_step': first['bytes'], 'world': world, 'grad_allreduce_bytes': red.flat.numel() * 4}


def _worker(rank, world, port, steps, warmup, q):
    try:
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group('nccl' if world > 1 else 'gloo', rank=rank, world_size=world)
        out = {mode: _run(rank, world, mode == 'sync', steps, warmup) for mode in ('unsync', 'sync', 'unsync_again')}
        dist.destroy_process_group()
        q.put((rank, out))
    except BaseException:
        q.put((rank, traceback.format_exc()))


def _world_run(world, steps, warmup):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, world, port, steps, warmup, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=1800) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(world):
        if not isinstance(got[r], dict):
            raise RuntimeError('rank %d failed:\n%s' % (r, got[r]))
    return got[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--world', type=int, default=None, help='ranks of the multi-GPU run (default: every visible GPU)')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('sync_stats_bench: no CUDA device (the numbers are GPU timings; there is no CPU mode)')
    props = torch.cuda.get_device_properties(0)
    res = {'device': props.name, 'gpus_visible': torch.cuda.device_count(), 'shape': 'retina_unet 3D, batch_norm, 2 x 128 x 128 x 64 per GPU',
           'steps': a.steps, 'warmup': a.warmup, 'world1': _world_run(1, a.steps, a.warmup)}
    try:
        import subprocess
        res['nvidia_smi'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the query is informational
        res['nvidia_smi'] = 'unavailable: %s' % e
    world = a.world or torch.cuda.device_count()
    res['worldN'] = _world_run(world, a.steps, a.warmup) if world > 1 else 'not measured: %d GPU visible' % torch.cuda.device_count()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
