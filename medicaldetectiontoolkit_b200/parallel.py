"""Data-parallel training: one process per GPU, ONE all-reduce per step over a flat fp32 gradient buffer (SURVEY.md §8e), and the opt-in
exchange of batch statistics (sync_batch_statistics) that gives each step the one-GPU batch.

The reference has no multi-GPU code (exec.py:38 is single-device).  The path shards by patch; without sync_batch_statistics the only
exchange is the gradient sum.  All parameter .grad tensors are views into one contiguous buffer, so backward accumulates straight into
the message and the averaged result is what the (fused) Adam reads — no flatten/unflatten copies.  Parameters that never receive a
gradient (Fpn.P1_conv2.*, backbone.py:175) still sit in the buffer as zeros, which keeps the bucket list static across ranks.
"""
import torch
import torch.distributed as dist


def _world(group):
    return dist.get_world_size(group), dist.get_rank(group)


def row_slots(n, k, device, group=None, dtype=torch.float64):
    """-> (buf, slot): a [world, n, k] exchange buffer filled with -0.0 and this rank's [n, k] slot in it, for a kernel to write into directly
    before all_reduce_rows(buf).  On the GPU the fill is the library's (mdt_exchange_fill), so the exchange adds no torch kernel."""
    world, rank = _world(group)
    device = torch.device(device)
    if device.type != 'cuda':
        buf = torch.full((world, n, k), -0.0, dtype=dtype, device=device)
        return buf, buf[rank]
    from . import _lib as L
    if dtype not in (torch.float64, torch.float32):
        raise ValueError("row_slots: fp64 or fp32 rows, got %s" % dtype)
    buf = torch.empty((world, n, k), dtype=dtype, device=device)
    with torch.cuda.device(device):
        L.check(L.load().mdt_exchange_fill(L.ptr(buf), buf.numel(), int(dtype == torch.float64), L.stream_ptr()))
    return buf, buf[rank]


def all_reduce_rows(buf, group=None):
    """[world, n, k] buffer whose slots each rank filled -> [world * n, k] in rank-major order.  One all_reduce(SUM): every other rank's copy
    of a slot holds -0.0, and v + (-0.0) is v for every v (signed zeros included), so each row arrives with its bits.  No host
    synchronisation.  A group of one rank has nothing to exchange: the buffer is already the result."""
    if buf.shape[0] > 1:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    return buf.view(buf.shape[0] * buf.shape[1], buf.shape[2])


def gather_rows(local, group=None):
    """fp64 [n, k] rows of this rank -> [world * n, k] of every rank, rank-major (the same n on every rank)"""
    if local.dtype != torch.float64 or local.dim() != 2:
        raise ValueError("gather_rows: expected fp64 [n, k] rows, got %s %s" % (local.dtype, tuple(local.shape)))
    buf, slot = row_slots(local.shape[0], local.shape[1], local.device, group)
    slot.copy_(local)
    return all_reduce_rows(buf, group)


_SHAPE_SLOTS = 8


def check_equal_batches(shape, device, group=None):
    """Every rank passes its input shape; raises RuntimeError on every rank unless all shapes are equal.  One tiny collective and one host read.
    The synchronised statistics assume the same per-rank batch: a rank with fewer samples would issue the same collectives over rows of another
    size, which mismatch or hang."""
    if dist.get_world_size(group) == 1:
        return
    shape = [int(v) for v in shape]
    if len(shape) > _SHAPE_SLOTS - 1:
        raise ValueError("check_equal_batches: at most %d dimensions" % (_SHAPE_SLOTS - 1))
    row = torch.full((1, _SHAPE_SLOTS), -1.0, dtype=torch.float64)
    row[0, 0] = len(shape)
    row[0, 1:1 + len(shape)] = torch.tensor(shape, dtype=torch.float64)
    rows = gather_rows(row.to(device), group).cpu()
    if not bool((rows == rows[:1]).all()):
        got = [tuple(int(v) for v in r[1:1 + int(r[0])]) for r in rows]
        raise RuntimeError("synchronised batch statistics need the same input shape on every rank, got %s (by rank)" % (got,))


def _roi_head_modules(net):
    """modules of the Mask R-CNN / UFRCNN+ RoI heads: their batches are RoI chunks whose count differs per rank, so they stay per rank"""
    from .mrcnn import Classifier, Mask
    skip = set()
    for m in net.modules():
        if isinstance(m, (Classifier, Mask)):
            skip.update(id(x) for x in m.modules())
    return skip


def sync_batch_statistics(net, group=None):
    """Opt in to the one-GPU batch under data parallelism: in training mode, the native batch norms of `net` (except the RoI heads') normalise
    over the whole batch of all ranks of `group` (None: the default group), and the Retina U-Net / UFRCNN+ / Detection U-Net seg losses take
    their dice and cross-entropy over it.  Returns `net`.

    Ranks must train on the same per-rank batch shape: a forward pre-hook on the backbone exchanges the input shape once per training forward
    and raises RuntimeError on every rank if they differ, before any statistics are exchanged.  In eval mode (validation, Predictor) every
    exchange is off, so ranks with unequal shards cannot hang; validation losses are then per rank."""
    from .backbone import FPN
    from .norm import _NativeBatchNorm
    if not dist.is_initialized():
        raise RuntimeError("sync_batch_statistics: no process group is initialised")
    group = group if group is not None else dist.group.WORLD
    skip = _roi_head_modules(net)
    for m in net.modules():
        if isinstance(m, _NativeBatchNorm) and id(m) not in skip:
            m.process_group = group
    backbones = [m for m in net.children() if isinstance(m, FPN)]
    if len(backbones) != 1:
        raise RuntimeError("sync_batch_statistics: expected one FPN backbone in %s, found %d" % (type(net).__name__, len(backbones)))

    def _check(module, args):
        if module.training:
            check_equal_batches(args[0].shape, args[0].device, group)

    if getattr(net, '_sync_hook', None) is not None:
        net._sync_hook.remove()
    net._sync_hook = backbones[0].register_forward_pre_hook(_check)
    net.sync_group = group
    return net


class FlatGradAllReduce(object):
    def __init__(self, module, world_size, group=None):
        self.world = world_size
        self.group = group
        params = [p for p in module.parameters() if p.requires_grad]
        n = sum(p.numel() for p in params)
        self.flat = torch.zeros(n, dtype=torch.float32, device=params[0].device)
        off = 0
        for p in params:
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            off += p.numel()
        self.params = params

    def zero_grad(self):
        self.flat.zero_()

    def _check_aliasing(self):
        """`optimizer.zero_grad()` (set_to_none=True by default) or any `p.grad = None` silently detaches a parameter from the flat buffer; the
        all-reduce would then average a stale buffer and the replicas diverge.  Re-bind (and carry over) such gradients."""
        base = self.flat.data_ptr()
        off = 0
        for p in self.params:
            want = base + off * 4
            if p.grad is None:                                  # released by zero_grad(set_to_none=True) and not produced since: contributes 0
                p.grad = self.flat[off:off + p.numel()].view_as(p)
                p.grad.zero_()
            elif p.grad.data_ptr() != want:
                view = self.flat[off:off + p.numel()].view_as(p)
                view.copy_(p.grad)
                p.grad = view
            off += p.numel()

    def all_reduce(self):
        self._check_aliasing()
        if self.world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
            self.flat.mul_(1.0 / self.world)
