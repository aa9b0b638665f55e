"""Instance norm, batch norm and leaky ReLU on libmdt_b200 (csrc/norm_act.cu) — the `norm` and `relu` options of NDConvGenerator
(utils/model_utils.py:739-781: nn.InstanceNorm{2,3}d, nn.BatchNorm{2,3}d, nn.LeakyReLU(inplace=True)).

The modules subclass torch's, so parameters, buffers (`weight`, `bias`, `running_mean`, `running_var`, `num_batches_tracked`), state-dict keys,
load_state_dict, train() / eval() and isinstance checks are exactly the reference's.  Only `forward` differs: one statistics pass and one
apply pass that also runs the following activation (and, inside a ResBlock, the residual add), all on channels-last maps.  Options the conv
factory never builds raise instead of running on a torch kernel; there is no CPU fallback.

A batch norm with `process_group` set (parallel.sync_batch_statistics) takes its training-mode statistics over the batch of all the group's
ranks: per-sample fp64 sums, one exchange of those rows, and the statistics added up in rank order (the same bits at any world size).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import parallel as P
from .conv import _workspace

ACTS = {None: 0, 'relu': 1, 'leaky_relu': 2}
LEAKY_SLOPE = 0.01   # nn.LeakyReLU's default, the factory's only slope


def _cl(t):
    """t with its channels innermost in memory ([N, S, C] for the kernels); any start offset is accepted"""
    fmt = torch.channels_last_3d if t.dim() == 5 else torch.channels_last if t.dim() == 4 else torch.contiguous_format
    return t.contiguous(memory_format=fmt), fmt


class _NormActFn(torch.autograd.Function):
    """y = act((x - mean) * rstd * weight + bias (+ residual)); batch statistics (and the running-statistics update) or running statistics"""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, num_batches_tracked, per_sample, batch_stats, momentum, eps, act):
        lib = L.load()
        L.require_cuda(x, weight, bias, residual, running_mean, running_var)
        x, fmt = _cl(x)
        if residual is not None:
            residual = residual.contiguous(memory_format=fmt)
        n, c = x.shape[0], x.shape[1]
        s = x[0, 0].numel()
        groups = n * c if per_sample else c
        mean = torch.empty(groups, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        y = torch.empty_like(x, memory_format=fmt)
        slope = LEAKY_SLOPE
        with torch.cuda.device(x.device):
            if batch_stats:
                ws = _workspace(lib.mdt_norm_workspace_bytes(n, s, c, int(per_sample)), x.device)
                L.check(lib.mdt_norm_stats(L.ptr(x), n, s, c, int(per_sample), eps, momentum, L.ptr(mean), L.ptr(rstd), L.ptr(running_mean),
                                           L.ptr(running_var), L.ptr(num_batches_tracked), L.ptr(ws), ws.numel(), L.stream_ptr()))
            else:
                L.check(lib.mdt_norm_eval_stats(L.ptr(running_mean), L.ptr(running_var), c, eps, L.ptr(mean), L.ptr(rstd), L.stream_ptr()))
            L.check(lib.mdt_norm_apply(L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(weight), L.ptr(bias), L.ptr(residual), n, s, c, int(per_sample),
                                       ACTS[act], slope, L.ptr(y), L.stream_ptr()))
        ctx.save_for_backward(x, y if act is not None else None, mean, rstd, weight)
        ctx.cfg = (fmt, per_sample, batch_stats, act, bias is not None, residual is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = L.load()
        x, y, mean, rstd, weight = ctx.saved_tensors
        fmt, per_sample, batch_stats, act, has_bias, has_res = ctx.cfg
        dy = dy.contiguous(memory_format=fmt)
        n, c = x.shape[0], x.shape[1]
        s = x[0, 0].numel()
        dx = torch.empty_like(x, memory_format=fmt)
        dw = torch.empty(c, dtype=torch.float32, device=x.device) if weight is not None and ctx.needs_input_grad[1] else None
        db = torch.empty(c, dtype=torch.float32, device=x.device) if has_bias and ctx.needs_input_grad[2] else None
        dres = torch.empty_like(x, memory_format=fmt) if has_res and ctx.needs_input_grad[3] else None
        with torch.cuda.device(x.device):
            ws = _workspace(lib.mdt_norm_workspace_bytes(n, s, c, int(per_sample)), x.device)
            L.check(lib.mdt_norm_backward(L.ptr(dy), L.ptr(y), L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(weight), n, s, c, int(per_sample), ACTS[act],
                                          LEAKY_SLOPE, int(batch_stats), L.ptr(dx), L.ptr(dw), L.ptr(db), L.ptr(dres), L.ptr(ws), ws.numel(),
                                          L.stream_ptr()))
        return dx, dw, db, dres, None, None, None, None, None, None, None, None


class _SyncBatchNormActFn(torch.autograd.Function):
    """_NormActFn for batch norm in training mode with the batch split across the ranks of `group`: per-sample sums -> one exchange ->
    statistics of the whole batch, and the same for the backward.  Every rank must pass the same n."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, num_batches_tracked, momentum, eps, act, group):
        lib = L.load()
        L.require_cuda(x, weight, bias, residual, running_mean, running_var)
        x, fmt = _cl(x)
        if residual is not None:
            residual = residual.contiguous(memory_format=fmt)
        n, c = x.shape[0], x.shape[1]
        s = x[0, 0].numel()
        mean = torch.empty(c, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        y = torch.empty_like(x, memory_format=fmt)
        with torch.cuda.device(x.device):
            ws = _workspace(lib.mdt_norm_sample_workspace_bytes(n, s, c), x.device)
            buf, slot = P.row_slots(n, 2 * c, x.device, group)
            L.check(lib.mdt_norm_sample_sums(L.ptr(x), n, s, c, L.ptr(slot), L.ptr(ws), ws.numel(), L.stream_ptr()))
            rows = P.all_reduce_rows(buf, group)
            L.check(lib.mdt_norm_stats_from_sums(L.ptr(rows), rows.shape[0], s, c, eps, momentum, L.ptr(mean), L.ptr(rstd), L.ptr(running_mean),
                                                 L.ptr(running_var), L.ptr(num_batches_tracked), L.stream_ptr()))
            L.check(lib.mdt_norm_apply(L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(weight), L.ptr(bias), L.ptr(residual), n, s, c, 0, ACTS[act],
                                       LEAKY_SLOPE, L.ptr(y), L.stream_ptr()))
        ctx.save_for_backward(x, y if act is not None else None, mean, rstd, weight)
        ctx.cfg = (fmt, act, bias is not None, residual is not None, group)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = L.load()
        x, y, mean, rstd, weight = ctx.saved_tensors
        fmt, act, has_bias, has_res, group = ctx.cfg
        dy = dy.contiguous(memory_format=fmt)
        n, c = x.shape[0], x.shape[1]
        s = x[0, 0].numel()
        dx = torch.empty_like(x, memory_format=fmt)
        dw = torch.empty(c, dtype=torch.float32, device=x.device) if weight is not None and ctx.needs_input_grad[1] else None
        db = torch.empty(c, dtype=torch.float32, device=x.device) if has_bias and ctx.needs_input_grad[2] else None
        dres = torch.empty_like(x, memory_format=fmt) if has_res and ctx.needs_input_grad[3] else None
        with torch.cuda.device(x.device):
            ws = _workspace(lib.mdt_norm_sample_workspace_bytes(n, s, c), x.device)
            buf, slot = P.row_slots(n, 2 * c, x.device, group)
            L.check(lib.mdt_norm_backward_sample_sums(L.ptr(dy), L.ptr(y), L.ptr(x), L.ptr(mean), L.ptr(rstd), n, s, c, ACTS[act], LEAKY_SLOPE,
                                                      L.ptr(slot), L.ptr(ws), ws.numel(), L.stream_ptr()))
            rows = P.all_reduce_rows(buf, group)
            L.check(lib.mdt_norm_backward_from_sums(L.ptr(dy), L.ptr(y), L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(weight), L.ptr(rows), rows.shape[0],
                                                    P.dist.get_rank(group) * n, n, s, c, ACTS[act], LEAKY_SLOPE, L.ptr(dx), L.ptr(dw), L.ptr(db),
                                                    L.ptr(dres), L.ptr(ws), ws.numel(), L.stream_ptr()))
        return dx, dw, db, dres, None, None, None, None, None, None, None


class _ActFn(torch.autograd.Function):
    """standalone activation; the backward reads the saved output (torch's rule for in-place activations)"""

    @staticmethod
    def forward(ctx, x, act, slope):
        lib = L.load()
        L.require_cuda(x)
        if x.dtype != torch.float32:
            raise L.MdtError("libmdt_b200 activations take float32 tensors only, got %s" % x.dtype)
        fmts = (torch.contiguous_format, torch.channels_last_3d if x.dim() == 5 else torch.channels_last if x.dim() == 4 else None)
        if not any(f is not None and x.is_contiguous(memory_format=f) for f in fmts):
            x = x.contiguous()
        y = torch.empty_like(x)   # dense input: the same strides, so the elementwise pass can run over raw memory
        with torch.cuda.device(x.device):
            L.check(lib.mdt_act_forward(L.ptr(x), x.numel(), ACTS[act], slope, L.ptr(y), L.stream_ptr()))
        ctx.save_for_backward(y)
        ctx.cfg = (act, slope)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = L.load()
        (y,) = ctx.saved_tensors
        act, slope = ctx.cfg
        if dy.stride() != y.stride():
            dy = torch.empty_like(y).copy_(dy)
        dx = torch.empty_like(y)
        with torch.cuda.device(y.device):
            L.check(lib.mdt_act_backward(L.ptr(dy), L.ptr(y), y.numel(), ACTS[act], slope, L.ptr(dx), L.stream_ptr()))
        return dx, None, None


def leaky_relu(x, negative_slope=LEAKY_SLOPE):
    return _ActFn.apply(x, 'leaky_relu', float(negative_slope))


class LeakyReLU(nn.LeakyReLU):
    """nn.LeakyReLU on the library's elementwise kernel.  `inplace` is kept for the module surface; the result is a new tensor."""

    def forward(self, input):
        return leaky_relu(input, self.negative_slope)


class _NativeNorm:
    """shared forward of the norm subclasses.  `act` is the activation the factory puts after the norm ('relu', 'leaky_relu' or None): it
    runs in the apply pass, and the slot after the norm holds a parameter-free marker."""

    act = None

    def _check_options(self, momentum, dtype):
        if momentum is None:
            raise ValueError("%s: momentum=None (cumulative moving average) is not supported by the native kernels" % type(self).__name__)
        if dtype not in (None, torch.float32):
            raise ValueError("%s: only float32 is supported by the native kernels, got %s" % (type(self).__name__, dtype))

    def norm_act(self, input, residual=None, act=None):
        """act(norm(input) (+ residual)) in one apply pass"""
        self._check_input_dim(input)
        if input.dim() != self._batched_dim:
            raise ValueError("%s: expected a batched %dD input, got %dD" % (type(self).__name__, self._batched_dim, input.dim()))
        if input.dtype != torch.float32:
            raise ValueError("%s: only float32 input is supported by the native kernels, got %s" % (type(self).__name__, input.dtype))
        if input.shape[1] != self.num_features:
            raise ValueError("expected input's size at dim=1 to match num_features (%d), but got: %d." % (self.num_features, input.shape[1]))
        if act not in ACTS:
            raise ValueError("unsupported activation %r" % (act,))
        if isinstance(self, nn.modules.instancenorm._InstanceNorm):
            F._verify_spatial_size(input.size())
            return _NormActFn.apply(input, None, None, residual, None, None, None, True, True, self.momentum, self.eps, act)
        batch_stats = self.training
        if batch_stats and self.process_group is not None:
            return _SyncBatchNormActFn.apply(input, self.weight, self.bias, residual, self.running_mean, self.running_var, self.num_batches_tracked,
                                             self.momentum, self.eps, act, self.process_group)
        if batch_stats:
            F._verify_batch_size(input.size())
        return _NormActFn.apply(input, self.weight, self.bias, residual, self.running_mean, self.running_var,
                                self.num_batches_tracked if batch_stats else None, False, batch_stats, self.momentum, self.eps, act)

    def forward(self, input, residual=None):
        return self.norm_act(input, residual, self.act)


class _NativeInstanceNorm(_NativeNorm):
    def _init_check(self, affine, track_running_stats, momentum, dtype):
        if affine or track_running_stats:
            raise ValueError("%s: affine / track_running_stats are not supported by the native kernels (the conv factory builds neither)"
                             % type(self).__name__)
        self._check_options(momentum, dtype)


class InstanceNorm3d(_NativeInstanceNorm, nn.InstanceNorm3d):
    _batched_dim = 5

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=False, track_running_stats=False, device=None, dtype=None):
        self._init_check(affine, track_running_stats, momentum, dtype)
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device, dtype)


class InstanceNorm2d(_NativeInstanceNorm, nn.InstanceNorm2d):
    _batched_dim = 4

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=False, track_running_stats=False, device=None, dtype=None):
        self._init_check(affine, track_running_stats, momentum, dtype)
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device, dtype)


class _NativeBatchNorm(_NativeNorm):
    # set by parallel.sync_batch_statistics: in training mode the statistics are then those of the whole batch across the group's ranks
    process_group = None

    def _init_check(self, affine, track_running_stats, momentum, dtype):
        if not (affine and track_running_stats):
            raise ValueError("%s: affine=False / track_running_stats=False are not supported by the native kernels (the conv factory builds "
                             "neither)" % type(self).__name__)
        self._check_options(momentum, dtype)


class BatchNorm3d(_NativeBatchNorm, nn.BatchNorm3d):
    _batched_dim = 5

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, device=None, dtype=None):
        self._init_check(affine, track_running_stats, momentum, dtype)
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device, dtype)


class BatchNorm2d(_NativeBatchNorm, nn.BatchNorm2d):
    _batched_dim = 4

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, device=None, dtype=None):
        self._init_check(affine, track_running_stats, momentum, dtype)
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device, dtype)
