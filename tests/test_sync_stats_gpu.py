"""Batch statistics across data-parallel ranks (parallel.sync_batch_statistics) on the GPU.

The entry points run through poisoned exact-size buffers; a sample's sums must have the same bits in a batch of 1, 2 or 5.  World 2 (gloo, both
ranks on cuda:0; also NCCL on cuda:0 / cuda:1 when two GPUs are visible) with one sample per rank is compared with world 1 on the two-sample
batch, both synchronised: batch-norm outputs, dx, statistics and running statistics, the seg-loss terms and sums must be bit-identical, and
per-rank seg-loss gradients exactly twice world 1's (each rank's loss holds the global term, and its gradient is summed over the ranks)."""
import ctypes
import datetime
import os
import socket
import sys
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
import torch.nn.functional as F

from _guarded import DEV, _run_guarded

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN_CASES = [((8, 8, 6), 18), ((8, 8, 6), 36), ((4, 4, 2), 576), ((32, 32, 16), 36), ((16, 12), 18), ((16, 12), 576)]
SEG_CASES = [(2, (64, 64, 32)), (3, (40, 24))]


def _lib():
    from medicaldetectiontoolkit_b200 import _lib as L
    return L, L.load()


def _err(a, b):
    return float((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------------------------ entry points
@pytest.mark.parametrize("n,s,c", [(1, 7, 3), (2, 384, 18), (5, 16384, 36), (3, 96, 576), (1, 300000, 18)])
def test_norm_sample_sums_guarded_and_batch_independent(n, s, c):
    L, lib = _lib()
    x = (torch.randn(5, s, c, device=DEV) * 3 + 1).contiguous()
    wsb = lib.mdt_norm_sample_workspace_bytes(n, s, c)
    got = _run_guarded(lambda o, ws: lib.mdt_norm_sample_sums(L.ptr(x), n, s, c, o[0], ws, wsb, L.stream_ptr()), [n * c * 16], wsb)
    rows = got[0].view(torch.float64).view(n, c, 2)
    ref = x[:n].double()
    assert torch.allclose(rows[..., 0], ref.sum(1), rtol=1e-12, atol=1e-9)
    assert torch.allclose(rows[..., 1], (ref * ref).sum(1), rtol=1e-12, atol=1e-9)
    # each sample of a batch of 5 has the bits it has alone, and a batch of 2 the bits of the batch of 5's first two
    def sums(xs):
        out = torch.empty(xs.shape[0], c, 2, dtype=torch.float64, device=DEV)
        ws = torch.empty(lib.mdt_norm_sample_workspace_bytes(xs.shape[0], s, c), dtype=torch.uint8, device=DEV)
        L.check(lib.mdt_norm_sample_sums(L.ptr(xs), xs.shape[0], s, c, L.ptr(out), L.ptr(ws), ws.numel(), L.stream_ptr()))
        return out
    five = sums(x)
    assert torch.equal(five[:n], rows) and torch.equal(sums(x[:2].contiguous()), five[:2])
    for j in range(5):
        assert torch.equal(sums(x[j:j + 1].contiguous())[0], five[j]), j
    # the backward sums, through guarded buffers, are batch-independent too
    dy, y = torch.randn_like(x), torch.randn_like(x)
    mean, rstd = torch.randn(c, device=DEV), torch.rand(c, device=DEV) + 0.5
    gb = _run_guarded(lambda o, ws: lib.mdt_norm_backward_sample_sums(L.ptr(dy), L.ptr(y), L.ptr(x), L.ptr(mean), L.ptr(rstd), n, s, c, 2, 0.01, o[0],
                                                                     ws, wsb, L.stream_ptr()), [n * c * 16], wsb)
    one = torch.empty(1, c, 2, dtype=torch.float64, device=DEV)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=DEV)
    L.check(lib.mdt_norm_backward_sample_sums(L.ptr(dy), L.ptr(y), L.ptr(x), L.ptr(mean), L.ptr(rstd), 1, s, c, 2, 0.01, L.ptr(one), L.ptr(ws),
                                              ws.numel(), L.stream_ptr()))
    assert torch.equal(one[0], gb[0].view(torch.float64).view(n, c, 2)[0])


def test_norm_from_sums_guarded():
    L, lib = _lib()
    n, s, c, N = 2, 384, 18, 4
    x, dy, res_y = (torch.randn(n, s, c, device=DEV) for _ in range(3))
    rows = torch.randn(N, c, 2, dtype=torch.float64, device=DEV).abs() * 100
    rm, rv = torch.randn(c, device=DEV), torch.rand(c, device=DEV) + 0.5
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)

    def stats(o, ws):
        r = [rm.clone(), rv.clone()]
        return lib.mdt_norm_stats_from_sums(L.ptr(rows), N, s, c, 1e-5, 0.1, o[0], o[1], L.ptr(r[0]), L.ptr(r[1]), L.ptr(nbt), L.stream_ptr())
    mean, rstd = (t.view(torch.float32) for t in _run_guarded(stats, [c * 4, c * 4], None))
    tot = rows.sum(0)
    mu = tot[:, 0] / (N * s)
    assert _err(mean, mu) < 1e-6 and _err(rstd, 1 / torch.sqrt((tot[:, 1] / (N * s) - mu * mu).clamp_min(0) + 1e-5)) < 1e-6
    wsb = lib.mdt_norm_sample_workspace_bytes(n, s, c)
    gamma = torch.randn(c, device=DEV)
    outs = _run_guarded(lambda o, ws: lib.mdt_norm_backward_from_sums(L.ptr(dy), L.ptr(res_y), L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(gamma),
                                                                     L.ptr(rows), N, 1, n, s, c, 2, 0.01, o[0], o[1], o[2], o[3], ws, wsb,
                                                                     L.stream_ptr()), [n * s * c * 4, c * 4, c * 4, n * s * c * 4], wsb)
    dgamma, dbeta = outs[1].view(torch.float32), outs[2].view(torch.float32)
    assert torch.equal(dgamma, rows[1:3, :, 1].sum(0).float()) and torch.equal(dbeta, rows[1:3, :, 0].sum(0).float())
    # argument errors come back as codes
    f = ctypes.c_void_p(0)
    assert lib.mdt_norm_sample_sums(f, 1, s, c, L.ptr(rows), L.ptr(rows), 1 << 20, L.stream_ptr()) == -1
    assert lib.mdt_norm_sample_sums(L.ptr(x), 0, s, c, L.ptr(rows), L.ptr(rows), 1 << 20, L.stream_ptr()) == -1
    assert lib.mdt_norm_sample_sums(L.ptr(x), 1, s, c, L.ptr(rows), L.ptr(rows), 16, L.stream_ptr()) == -2
    assert lib.mdt_norm_stats_from_sums(L.ptr(rows), 0, s, c, 1e-5, 0.1, L.ptr(x), L.ptr(x), f, f, f, L.stream_ptr()) == -1
    assert lib.mdt_norm_backward_from_sums(L.ptr(dy), f, L.ptr(x), L.ptr(mean), L.ptr(rstd), f, L.ptr(rows), N, 3, n, s, c, 0, 0.01, L.ptr(x), f, f, f,
                                           L.ptr(rows), 1 << 20, L.stream_ptr()) == -1
    assert lib.mdt_norm_backward_from_sums(L.ptr(dy), f, L.ptr(x), L.ptr(mean), L.ptr(rstd), f, L.ptr(rows), N, 0, n, s, c, 0, 0.01, L.ptr(x), f, f, f,
                                           L.ptr(rows), 8, L.stream_ptr()) == -2
    assert lib.mdt_norm_sample_workspace_bytes(0, s, c) == 0


def _seg_inputs(n, sp, c, seed):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn((n, c) + sp, generator=g) * 3).to(DEV)
    seg = torch.randint(0, c, (n,) + sp, generator=g, dtype=torch.uint8).to(DEV)
    return logits, seg


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("c", [2, 3, 8])
def test_seg_sample_sums_guarded_and_batch_independent(weighted, c):
    L, lib = _lib()
    logits, seg = _seg_inputs(5, (40, 24, 12), c, 1)
    vox, nv = 40 * 24 * 12, 3 * c + 1
    lay = L.i64arr(logits.stride()[:2] + (1,))
    w = torch.rand(c, device=DEV) + 0.5

    def call(nb, o, ws, wsb):
        if weighted:
            return lib.mdt_seg_loss_weighted_sample_sums(L.ptr(logits), lay, L.ptr(seg), nb, vox, c, L.ptr(w), o, ws, wsb, L.stream_ptr())
        return lib.mdt_seg_loss_sample_sums(L.ptr(logits), lay, L.ptr(seg), nb, vox, c, o, ws, wsb, L.stream_ptr())
    rows = {}
    for nb in (1, 2, 5):
        wsb = lib.mdt_seg_loss_sample_workspace_bytes(nb, vox, c)
        rows[nb] = _run_guarded(lambda o, ws: call(nb, o[0], ws, wsb), [nb * nv * 8], wsb)[0].view(torch.float64).view(nb, nv)
    assert torch.equal(rows[1], rows[5][:1]) and torch.equal(rows[2], rows[5][:2])
    # against fp64 torch, per sample
    p = torch.softmax(logits.double(), 1).flatten(2)
    oh = F.one_hot(seg.long().flatten(1), c).movedim(-1, 1).double()
    nll = -torch.log_softmax(logits.double(), 1).flatten(2).gather(1, seg.long().flatten(1)[:, None])[:, 0]
    wt = w.double()[seg.long().flatten(1)] if weighted else torch.ones_like(nll)
    ref = torch.cat([(p * oh).sum(2), p.sum(2), oh.sum(2), (wt * nll).sum(1, keepdim=True)], 1)
    assert _err(rows[5], ref) < 1e-6
    # from-sums and the global backward through guarded buffers
    wp = w if weighted else None
    sums_out = _run_guarded(lambda o, ws: lib.mdt_seg_loss_from_sums(L.ptr(rows[5]), 5, vox, c, 1.0, 1e-6, L.ptr(wp), o[0], o[1], L.stream_ptr()),
                            [nv * 8, 8], None)
    acc = rows[5][0].clone()
    for j in range(1, 5):
        acc = acc + rows[5][j]
    assert torch.equal(sums_out[0].view(torch.float64), acc)
    gout = torch.tensor([0.5, 0.25], device=DEV)
    sums = sums_out[0].view(torch.float64).clone()

    def bwd(o, ws):
        if weighted:
            return lib.mdt_seg_loss_weighted_backward_global(L.ptr(logits), lay, L.ptr(seg), 2, vox, c, 1.0, 1e-6, L.ptr(w), L.ptr(sums), 5 * vox,
                                                             L.ptr(gout), 1, o[0], L.stream_ptr())
        return lib.mdt_seg_loss_backward_global(L.ptr(logits), lay, L.ptr(seg), 2, vox, c, 1.0, 1e-6, L.ptr(sums), 5 * vox, L.ptr(gout), 1, o[0],
                                                L.stream_ptr())
    _run_guarded(bwd, [2 * c * vox * 4], None)
    # argument errors come back as codes
    f = ctypes.c_void_p(0)
    assert lib.mdt_seg_loss_sample_sums(f, lay, L.ptr(seg), 1, vox, c, L.ptr(sums), L.ptr(sums), 1 << 20, L.stream_ptr()) == -1
    assert lib.mdt_seg_loss_sample_sums(L.ptr(logits), lay, L.ptr(seg), 1, vox, 9, L.ptr(sums), L.ptr(sums), 1 << 20, L.stream_ptr()) == -3
    assert lib.mdt_seg_loss_sample_sums(L.ptr(logits), lay, L.ptr(seg), 1, vox, c, L.ptr(sums), L.ptr(sums), 8, L.stream_ptr()) == -2
    assert lib.mdt_seg_loss_weighted_sample_sums(L.ptr(logits), lay, L.ptr(seg), 1, vox, c, f, L.ptr(sums), L.ptr(sums), 1 << 20, L.stream_ptr()) == -1
    assert lib.mdt_seg_loss_from_sums(f, 1, vox, c, 1.0, 1e-6, f, L.ptr(sums), L.ptr(gout), L.stream_ptr()) == -1
    assert lib.mdt_seg_loss_backward_global(L.ptr(logits), lay, L.ptr(seg), 2, vox, c, 1.0, 1e-6, L.ptr(sums), vox, L.ptr(gout), 1, L.ptr(logits),
                                            L.stream_ptr()) == -1
    assert lib.mdt_seg_loss_backward_global(L.ptr(logits), lay, L.ptr(seg), 2, vox, c, 1.0, 1e-6, L.ptr(sums), 5 * vox, L.ptr(gout), 0, L.ptr(logits),
                                            L.stream_ptr()) == -1
    assert lib.mdt_exchange_fill(f, 4, 1, L.stream_ptr()) == -1
    assert lib.mdt_seg_loss_sample_workspace_bytes(1, vox, 9) == 0


# ------------------------------------------------------------------------------------------------------------------ world 2 vs world 1
def _bn_case(rank, world, sp, c, seed):
    from medicaldetectiontoolkit_b200 import norm as N
    import torch.distributed as dist
    g = torch.Generator().manual_seed(seed)
    full = [torch.randn((2, c) + sp, generator=g) * 2 + 0.5 for _ in range(3)]   # x, residual, dy of the whole batch
    n = 2 // world
    dev = torch.device('cuda', torch.cuda.current_device())
    x, res, dy = (t[rank * n:(rank + 1) * n].to(dev) for t in full)
    x.requires_grad_(True)
    res.requires_grad_(True)
    m = (N.BatchNorm3d(c) if len(sp) == 3 else N.BatchNorm2d(c)).to(dev)
    with torch.no_grad():
        m.weight.copy_(torch.randn(c, generator=g))
        m.bias.copy_(torch.randn(c, generator=g))
    m.process_group = dist.group.WORLD
    m.train()
    y = m.norm_act(x, residual=res, act='leaky_relu')
    mean, rstd = y.grad_fn.saved_tensors[2:4]
    y.backward(dy)
    out = dict(y=y, dx=x.grad, dres=res.grad, mean=mean, rstd=rstd, rm=m.running_mean, rv=m.running_var, nbt=m.num_batches_tracked,
               dgamma=m.weight.grad, dbeta=m.bias.grad)
    if world == 1:   # fp64 torch on the whole batch
        x64, r64 = x.detach().double().requires_grad_(True), res.detach().double().requires_grad_(True)
        w64, b64 = m.weight.detach().double().requires_grad_(True), m.bias.detach().double().requires_grad_(True)
        rm, rv = torch.zeros(c, dtype=torch.float64, device=dev), torch.ones(c, dtype=torch.float64, device=dev)
        y64 = F.leaky_relu(F.batch_norm(x64, rm, rv, w64, b64, True, 0.1, 1e-5) + r64, 0.01)
        y64.backward(dy.double())
        out['ref'] = dict(y=y64, dx=x64.grad, dres=r64.grad, dgamma=w64.grad, dbeta=b64.grad, rm=rm, rv=rv)
    return _cpu(out)


def _cpu(d):
    """host numpy copies (they cross the result queue by value: the worker may exit before the parent reads it)"""
    return {k: (_cpu(v) if isinstance(v, dict) else v.detach().cpu().numpy().copy()) for k, v in d.items()}


def _torch(d):
    def conv(v):
        if isinstance(v, dict):
            return _torch(v)
        if isinstance(v, list):
            return [conv(x) for x in v]
        return torch.from_numpy(v) if isinstance(v, np.ndarray) else v
    return {k: conv(v) for k, v in d.items()}


def _seg_case(rank, world, n_total, sp, c, weighted, seed):
    from medicaldetectiontoolkit_b200 import native_ops as NO
    import torch.distributed as dist
    dev = torch.device('cuda', torch.cuda.current_device())
    logits, seg = _seg_inputs(n_total, sp, c, seed)
    n = n_total // world
    lg = logits[rank * n:(rank + 1) * n].to(dev).contiguous(memory_format=torch.channels_last_3d if len(sp) == 3 else torch.channels_last)
    lg.requires_grad_(True)
    tg = seg[rank * n:(rank + 1) * n].to(dev).contiguous()
    w = (torch.arange(c, dtype=torch.float32, device=dev) + 1) / c if weighted else None
    dice, ce = NO.seg_loss(lg, tg, false_positive_weight=0.5, class_weights=w, group=dist.group.WORLD)
    sums = dice.grad_fn.saved_tensors[2].clone()
    (dice * 0.75 + ce).backward()
    out = dict(dice=dice, ce=ce, sums=sums, grad=lg.grad)
    if world == 1:
        p = torch.softmax(lg.detach().double(), 1)
        oh = F.one_hot(tg.long(), c).movedim(-1, 1).double()
        ax = tuple([0] + list(range(2, 2 + len(sp))))
        inter, psum, tsum = (p * oh).sum(ax), p.sum(ax), oh.sum(ax)
        dref = ((2 * inter + 1e-6) / (0.5 * psum + tsum + 1e-6))[1:].mean()
        ceref = F.cross_entropy(lg.detach().double(), tg.long(), weight=None if w is None else w.double())
        out['ref'] = dict(dice=dref, ce=ceref)
    return _cpu(out)


def _det_unet_case(rank, world, sync):
    """one train step of a batch-norm Detection U-Net (3D, 2 x 64 x 64 x 32) on this rank's share of the batch"""
    import torch.distributed as dist
    from medicaldetectiontoolkit_b200 import detection_unet, parallel
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    dev = torch.device('cuda', torch.cuda.current_device())
    cf = make_cf('detection_unet', 3, (64, 64, 32))
    cf.norm = 'batch_norm'
    torch.manual_seed(0)
    net = detection_unet.net(cf, None).to(dev)
    if sync:
        parallel.sync_batch_statistics(net)
    red = parallel.FlatGradAllReduce(net, world)
    full = synthetic_batch(cf, 2, seed=3)
    n = 2 // world
    batch = {k: (v[rank * n:(rank + 1) * n] if k in ('data', 'seg', 'bb_target', 'roi_labels') else v) for k, v in full.items()}
    net.train()
    red.zero_grad()
    seg_logits = net._logits(net._to_device(batch['data']))
    dice_loss, ce_loss = net.seg_loss_terms(seg_logits, net._to_device(batch['seg'], dtype=torch.uint8).contiguous())
    (dice_loss + ce_loss).backward()
    red.all_reduce()
    torch.cuda.synchronize()
    stats = {k: v.clone() for k, v in net.state_dict().items() if 'running' in k or 'num_batches' in k}   # later forwards move them on
    grads = {k: p.grad.clone() for k, p in net.named_parameters()}
    out = dict(logits=seg_logits, dice=dice_loss, ce=ce_loss, stats=stats, grads=grads)
    # eval mode issues no collective, and ranks may then hold batches of different sizes
    calls = [0]
    real = dist.all_reduce

    def counting(*a, **k):
        calls[0] += 1
        return real(*a, **k)
    dist.all_reduce = counting
    try:
        net.eval()
        with torch.no_grad():
            net.test_forward({'data': full['data'][:1 + rank]})
            lg = net._logits(net._to_device(full['data'][:1 + rank]))
            net.seg_loss_terms(lg, net._to_device(full['seg'][:1 + rank], dtype=torch.uint8).contiguous())
        torch.cuda.synchronize()
        out['eval_collectives'] = torch.tensor(calls[0])
        if sync:
            net.train()
            calls[0] = 0
            with torch.no_grad():
                net._logits(net._to_device(batch['data']))
            out['train_collectives'] = torch.tensor(calls[0])
            # unequal training batches: RuntimeError on every rank, before any statistics exchange
            try:
                with torch.no_grad():
                    net._logits(net._to_device(full['data'][:1 + rank]))
                out['mismatch_raised'] = torch.tensor(0)
            except RuntimeError as e:
                out['mismatch_raised'] = torch.tensor(int('same input shape' in str(e)))
    finally:
        dist.all_reduce = real
    return _cpu(out)


def _split(full, rank, world):
    n = 2 // world
    return {k: (v[rank * n:(rank + 1) * n] if k in ('data', 'seg', 'bb_target', 'roi_labels', 'roi_masks') else v) for k, v in full.items()}


def _retina_case(rank, world):
    """batch-norm Retina U-Net (3D 2 x 64 x 64 x 32): head logits, seg-loss terms and running statistics of this rank's share; then one whole
    train step (its SHEM draws differ per rank, so its anchor losses are not compared)"""
    from medicaldetectiontoolkit_b200 import parallel, retina_unet
    from medicaldetectiontoolkit_b200._detector import seg_loss_terms
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    dev = torch.device('cuda', torch.cuda.current_device())
    cf = make_cf('retina_unet', 3, (64, 64, 32))
    cf.norm = 'batch_norm'
    torch.manual_seed(0)
    net = parallel.sync_batch_statistics(retina_unet.net(cf, None).to(dev))
    red = parallel.FlatGradAllReduce(net, world)
    batch = _split(synthetic_batch(cf, 2, seed=4), rank, world)
    net.train()
    class_logits, pred_deltas, seg_logits = net._forward_logits(net._to_device(batch['data']))
    dice, ce = seg_loss_terms(seg_logits, net._seg_to_device(batch['seg'], True), cf, group=net.seg_loss_group())
    stats = {k: v.clone() for k, v in net.state_dict().items() if 'running' in k or 'num_batches' in k}
    out = dict(class_logits=class_logits, pred_deltas=pred_deltas, seg_logits=seg_logits, dice=dice, ce=ce, stats=stats)
    del class_logits, pred_deltas, seg_logits, dice, ce
    red.zero_grad()
    torch.manual_seed(1)
    res = net.train_forward(batch)
    res['torch_loss'].backward()
    red.all_reduce()
    torch.cuda.synchronize()
    out['step_loss'] = res['torch_loss'].detach()
    return _cpu(out)


def _mrcnn_case(rank, world):
    """batch-norm Mask R-CNN (3D 2 x 64 x 64 x 32) whose ranks split their proposals into different numbers of classifier chunks (roi_chunk_size
    64 on rank 0, 16 elsewhere: 2 and 8 chunks of 2 x 64 proposals): the step must complete; the backbone and RPN statistics are synchronised, the
    RoI heads' stay per rank"""
    from medicaldetectiontoolkit_b200 import mrcnn, parallel
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    dev = torch.device('cuda', torch.cuda.current_device())
    cf = make_cf('mrcnn', 3, (64, 64, 32))
    cf.norm, cf.relu = 'batch_norm', 'leaky_relu'
    cf.post_nms_rois_training = cf.post_nms_rois_inference = 64
    cf.pre_nms_limit = 1000
    cf.roi_chunk_size = 64 if rank == 0 else 16
    torch.manual_seed(0)
    net = parallel.sync_batch_statistics(mrcnn.net(cf, None).to(dev))
    red = parallel.FlatGradAllReduce(net, world)
    # two images per rank (with one, the per-rank RoI classifier can get a single RoI in the loss pass, which batch norm refuses); rank 1
    # trains on the inverted noise image, so unsynchronised backbone statistics would differ between the ranks
    batch = synthetic_batch(cf, 2, seed=2, with_masks=True)
    if rank == 1:
        batch['data'] = 1.0 - batch['data']
    net.train()
    red.zero_grad()
    torch.manual_seed(1)
    np.random.seed(1)
    res = net.train_forward(batch, monitor_anchors=False)
    res['torch_loss'].backward()
    red.all_reduce()
    torch.cuda.synchronize()
    stats = {k: v.clone() for k, v in net.state_dict().items() if 'running' in k or 'num_batches' in k}
    return _cpu(dict(stats=stats, loss=res['torch_loss'].detach(), chunks=torch.tensor(-(-2 * cf.post_nms_rois_training // cf.roi_chunk_size))))


def _profile_case(rank, world):
    """the CUDA kernels of one Detection U-Net seg-loss step without and with synchronisation (same net, same batch)"""
    from medicaldetectiontoolkit_b200 import detection_unet, parallel
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    dev = torch.device('cuda', torch.cuda.current_device())
    cf = make_cf('detection_unet', 3, (64, 64, 32))
    cf.norm = 'batch_norm'
    torch.manual_seed(0)
    net = detection_unet.net(cf, None).to(dev)
    batch = _split(synthetic_batch(cf, 2, seed=3), rank, world)
    net.train()

    def step():
        net.zero_grad(set_to_none=True)
        lg = net._logits(net._to_device(batch['data']))
        d, c = net.seg_loss_terms(lg, net._to_device(batch['seg'], dtype=torch.uint8).contiguous())
        (d + c).backward()
        torch.cuda.synchronize()

    def kernels():
        step()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step()
        return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    plain = kernels()
    parallel.sync_batch_statistics(net)
    synced = kernels()
    # copies and fills of the runtime are not compute kernels; the library's kernels live in namespace mdt
    extra = sorted(k for k in synced - plain if 'mdt::' not in k and not k.startswith(('Memcpy', 'Memset')))
    return {'extra': extra, 'synced_mdt': sorted(k for k in synced - plain if 'mdt::' in k)}


def _worker(rank, world, devices, backend, port, q):
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import torch.distributed as dist
        torch.cuda.set_device(torch.device(devices[rank]))
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        # a collective that another rank never issues fails after this timeout instead of waiting for the default 30 minutes
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
        res = {'bn': [_bn_case(rank, world, sp, c, 10 + i) for i, (sp, c) in enumerate(BN_CASES)],
               'seg': [_seg_case(rank, world, 2, sp, c, wt, 20 + i) for i, (c, sp) in enumerate(SEG_CASES) for wt in (False, True)],
               'dunet': _det_unet_case(rank, world, sync=True),
               'retina': _retina_case(rank, world)}
        if world == 2:
            res['dunet_nosync'] = _det_unet_case(rank, world, sync=False)
            res['mrcnn'] = _mrcnn_case(rank, world)
            res['profile'] = _profile_case(rank, world)
        dist.destroy_process_group()
        q.put((rank, res))
    except BaseException:
        q.put((rank, traceback.format_exc()))


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _spawn(devices, backend):
    world = len(devices)
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, devices, backend, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=900) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(world):
        assert isinstance(got[r], dict), 'rank {} failed:\n{}'.format(r, got[r])
    return [_torch(got[r]) for r in range(world)]


@pytest.fixture(scope='module')
def world1():
    return _spawn(['cuda:0'], 'gloo')[0]


@pytest.fixture(scope='module')
def world2_one_gpu():
    return _spawn(['cuda:0', 'cuda:0'], 'gloo')


def _cat(ranks, key, sub):
    return torch.cat([r[key][sub] if sub is not None else r[key] for r in ranks])


def _check_world2(w1, ranks):
    for i, (sp, c) in enumerate(BN_CASES):
        one, two = w1['bn'][i], [r['bn'][i] for r in ranks]
        for k in ('y', 'dx', 'dres'):
            assert torch.equal(torch.cat([t[k] for t in two]), one[k]), (sp, c, k)
        for k in ('mean', 'rstd', 'rm', 'rv', 'nbt'):
            for t in two:
                assert torch.equal(t[k], one[k]), (sp, c, k)
        for k in ('dgamma', 'dbeta'):   # each rank's share; FlatGradAllReduce adds them (and divides by the world size)
            assert _err(two[0][k] + two[1][k], one[k].double()) < 1e-6, (sp, c, k)
        ref = one['ref']
        assert _err(one['y'], ref['y']) < 4e-6 and _err(one['dx'], ref['dx']) < 1e-5 and _err(one['dres'], ref['dres']) < 1e-5, (sp, c)
        assert _err(one['dgamma'], ref['dgamma']) < 1e-5 and _err(one['dbeta'], ref['dbeta']) < 1e-5, (sp, c)
        assert _err(one['rm'], ref['rm']) < 1e-6 and _err(one['rv'], ref['rv']) < 1e-6, (sp, c)
    for i, one in enumerate(w1['seg']):
        two = [r['seg'][i] for r in ranks]
        for t in two:
            for k in ('dice', 'ce', 'sums'):
                assert torch.equal(t[k], one[k]), (i, k)
        n = one['grad'].shape[0] // 2
        for r, t in enumerate(two):   # 2x world 1's, bit for bit: a power-of-two scale is exact
            assert torch.equal(t['grad'], 2 * one['grad'][r * n:(r + 1) * n]), i
        assert abs(one['dice'].item() - one['ref']['dice'].item()) <= 1e-6 * abs(one['ref']['dice'].item()), i
        assert abs(one['ce'].item() - one['ref']['ce'].item()) <= 1e-6 * abs(one['ref']['ce'].item()), i
    one, two = w1['dunet'], [r['dunet'] for r in ranks]
    assert torch.equal(torch.cat([t['logits'] for t in two]), one['logits'])
    for t in two:
        assert torch.equal(t['dice'], one['dice']) and torch.equal(t['ce'], one['ce'])
        for k, v in one['stats'].items():
            assert torch.equal(t['stats'][k], v), k
        # the averaged gradients: relative L2 of the whole flat gradient, and per parameter against a floor of 1e-2 of the whole norm (a conv
        # bias feeding a batch norm has an analytically zero gradient; what it holds, ~1e-5 of the whole norm, is rounding noise)
        flat1 = torch.cat([v.double().flatten() for v in one['grads'].values()])
        flat2 = torch.cat([t['grads'][k].double().flatten() for k in one['grads']])
        assert float((flat2 - flat1).norm() / flat1.norm()) <= 1e-5
        for k, v in one['grads'].items():
            floor = max(float(v.double().norm()), 1e-2 * float(flat1.norm()))
            assert float((t['grads'][k].double() - v.double()).norm()) <= 1e-5 * floor, k
        assert int(t['eval_collectives']) == 0 and int(t['train_collectives']) > 0 and int(t['mismatch_raised']) == 1
    rone, two = w1['retina'], [r['retina'] for r in ranks]
    for k in ('class_logits', 'pred_deltas', 'seg_logits'):
        assert torch.equal(torch.cat([t[k] for t in two]), rone[k]), k
    for t in two:
        assert torch.equal(t['dice'], rone['dice']) and torch.equal(t['ce'], rone['ce'])
        for k, v in rone['stats'].items():
            assert torch.equal(t['stats'][k], v), k
        assert bool(torch.isfinite(t['step_loss']).all())
    m = [r['mrcnn'] for r in ranks]
    assert [int(t['chunks']) for t in m] == [2, 8] and all(bool(torch.isfinite(t['loss']).all()) for t in m)
    heads = [k for k in m[0]['stats'] if k.startswith(('classifier.', 'mask.'))]
    shared = [k for k in m[0]['stats'] if k.startswith(('fpn.', 'rpn.'))]
    assert heads and shared and len(heads) + len(shared) == len(m[0]['stats'])
    for k in shared:
        assert torch.equal(m[0]['stats'][k], m[1]['stats'][k]), k
    nbt = 'classifier.conv1.0.1.num_batches_tracked'
    assert [int(t['stats'][nbt]) for t in m] == [3, 9]     # once per chunk of the gradient-free pass, once in the loss pass
    assert not torch.equal(m[0]['stats']['classifier.conv1.0.1.running_mean'], m[1]['stats']['classifier.conv1.0.1.running_mean'])
    for r in ranks:
        assert not r['profile']['extra'], r['profile']['extra']
        assert any('sample' in k or 'from_sums' in k or 'neg_zero' in k for k in r['profile']['synced_mdt'])
    # negative control: without synchronisation world 2 is far from world 1
    free = [r['dunet_nosync'] for r in ranks]
    assert abs(free[0]['dice'].item() - one['dice'].item()) > 1e-4 * abs(one['dice'].item())
    assert float((torch.cat([t['logits'] for t in free]) - one['logits']).abs().max()) > 1e-4 * float(one['logits'].abs().max())
    assert int(free[0]['eval_collectives']) == 0


def test_world2_on_one_gpu_equals_world1(world1, world2_one_gpu):
    _check_world2(world1, world2_one_gpu)


def test_world2_nccl_on_two_gpus_equals_world1(world1):
    if torch.cuda.device_count() < 2:
        pytest.skip('one GPU visible: the NCCL world-2 run is unverified')
    _check_world2(world1, _spawn(['cuda:0', 'cuda:1'], 'nccl'))


# ------------------------------------------------------------------------------------------------------------------ Predictor, unequal shards
class _Log:
    def info(self, *a, **k):
        pass

    warning = info


def _predict_worker(rank, world, port, root, q):
    """a synchronised batch-norm Retina U-Net predicts a 3-patient toy test set over 2 ranks (shards of 2 and 1 patients): eval mode exchanges
    nothing, so the ranks' different numbers of forwards cannot hang"""
    try:
        sys.path.insert(0, ROOT)
        import pickle
        import shutil
        import torch.distributed as dist
        from medicaldetectiontoolkit_b200 import data_loader as D
        from medicaldetectiontoolkit_b200 import parallel, predictor, retina_unet
        torch.cuda.set_device(0)
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group('gloo', rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
        cf = _toy_cf(root)
        cf.fold_dir = os.path.join(root, 'run-r{}-w{}'.format(rank, world))
        shutil.copytree(os.path.join(root, 'checkpoints'), cf.fold_dir)
        net = parallel.sync_batch_statistics(retina_unet.net(cf, None).to('cuda:0'))
        gen = D.get_test_generator(cf, _Log(), rank, world)
        out = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(gen)
        torch.cuda.synchronize()
        dist.destroy_process_group()
        q.put((rank, {'n_test': gen['n_test'], 'results': None if out is None else pickle.dumps(out)}))
    except BaseException:
        q.put((rank, traceback.format_exc()))


def _toy_cf(root):
    from medicaldetectiontoolkit_b200.configs import make_cf
    cf = make_cf('retina_unet', 2, (320, 320), exp='toy_exp', batch_size=4)
    for k, v in dict(norm='batch_norm', test_aug=False, return_masks_in_test=False, wcs_iou=1e-5, fold=0, folds=[0], test_n_epochs=1,
                     model_min_confidence=0.0).items():
        setattr(cf, k, v)
    cf.pp_data_path = os.path.join(root, 'donuts_shape', 'train')
    cf.pp_test_data_path = os.path.join(root, 'donuts_shape', 'test')
    cf.exp_dir = root
    return cf


def test_predictor_over_unequal_shards_with_a_synchronised_net(tmp_path):
    from medicaldetectiontoolkit_b200 import generate_toys as G
    from medicaldetectiontoolkit_b200 import retina_unet
    root = str(tmp_path)
    G.generate_experiment(root, 'donuts_shape', 4, 3, 'donuts_shape', seed=9)
    torch.manual_seed(11)
    net = retina_unet.net(_toy_cf(root), None).to('cuda:0')
    os.makedirs(os.path.join(root, 'checkpoints', '0_best_checkpoint'))
    torch.save(net.state_dict(), os.path.join(root, 'checkpoints', '0_best_checkpoint', 'params.pth'))
    np.save(os.path.join(root, 'checkpoints', 'epoch_ranking.npy'), np.arange(1))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_predict_worker, args=(r, 2, port, root, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=600) for _ in range(2))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(2):
        assert isinstance(got[r], dict), 'rank {} failed:\n{}'.format(r, got[r])
    import pickle
    assert [got[r]['n_test'] for r in range(2)] == [2, 1]
    assert got[1]['results'] is None and len(pickle.loads(got[0]['results'])) == 3
