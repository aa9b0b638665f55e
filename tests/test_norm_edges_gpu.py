"""The instance-norm / batch-norm / activation kernels of csrc/norm_act.cu at the edges of their reduction split, every output against fp64 (GPU).

tests/test_norm_gpu.py checks these kernels through the modules of norm.py at the model's shapes.  Here every call goes through the C ABI with
guarded, poisoned exact-size buffers (tests/_guarded.py: base offsets 0 / 256 / 768, outputs poisoned, the workspace poisoned in one run and
zeroed in another, bit-identical outputs across runs), and every output is compared with an fp64 restatement:
  * the split matrix: shapes whose block split (tests/test_norm_split_model_cpu.py restates make_geo / make_sample_geo) reaches 1, 2-31, 32
    and 33 chunks per sample group, the chunk caps, a short last chunk, fewer rows per block than row lanes and channel counts around the
    256-lane passes; module-level assertions check that the case lists reach every one of those regimes;
  * every argument combination of mdt_norm_backward, mdt_norm_eval_stats, the synchronised-statistics entries (per-sample sums, statistics
    and backward from the exchanged rows), the activations past one grid-stride sweep;
  * values at the edges: a NaN or an Inf poisons exactly its group, constant groups, offset data, pre-activations exactly at 0.
Accuracy: e = max_i |got_i - ref_i| / mag_i, where mag_i is the same expression evaluated on absolute values (for rstd, on the terms of
E[x^2] - mean^2 + eps), so a kernel that drops one block's partial or hands it to the neighbouring channel fails by orders of magnitude
(test_metric_catches_a_planted_split_error).  The worst e per output is printed under -s.  NaN and Inf positions must equal the reference's."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_norm_split_model_cpu as M
from _guarded import DEV, _run_guarded
from medicaldetectiontoolkit_b200 import _lib as L

pytestmark = pytest.mark.gpu

EPS, MOM, SLOPE = 1e-5, 0.1, 0.01
EPS64 = float(np.float32(EPS))       # the kernels take eps as a float
F64 = torch.float64

_SPLIT, _SAMPLE = M.covered()
assert M.SPLIT_REGIMES <= _SPLIT, M.SPLIT_REGIMES - _SPLIT
assert M.SAMPLE_REGIMES <= _SAMPLE, M.SAMPLE_REGIMES - _SAMPLE

# Bounds on e (see the module docstring): 4x the worst value measured over every case of this file on an H100 80GB HBM3 (power limit 700 W),
# the measured value beside each.  The fp64 sums of exactly representable terms (x, x^2, g) get a bound of a few fp64 ulps instead.  A block's
# partial dropped or handed to the neighbouring channel gives e >= 3e-2 (test_metric_catches_a_planted_split_error).
TAU = {
    "mean": 2.3e-7,          # fp64 sums rounded to fp32; measured worst 5.60e-8
    "rstd": 2.3e-7,          # measured worst 5.64e-8
    "running_mean": 1.9e-7,  # measured worst 4.69e-8
    "running_var": 2.4e-7,   # measured worst 6.01e-8
    "y": 1.0e-6,             # fp32 (x - mean) * rstd * gamma + beta + residual; measured worst 2.53e-7
    "dx": 8.2e-7,            # measured worst 2.03e-7
    "dgamma": 4.1e-7,        # fp64 sums of fp32 g * xhat; measured worst 1.02e-7
    "dbeta": 1.9e-7,         # measured worst 4.80e-8
    "dres": 3.3e-7,          # fp32 dy * slope against fp64 (bit-exact against the fp32 rule); measured worst 8.10e-8
    "sums_x": 2e-15,         # measured worst 0
    "sums_x2": 2e-15,        # measured worst 4.26e-16
    "bsums_g": 2e-15,        # measured worst 3.49e-18
    "bsums_gx": 1.4e-7,      # fp32 xhat in the kernel; measured worst 3.51e-8
}
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst e per output:", {k: "%.3g" % v for k, v in sorted(_WORST.items())})


def _check(tag, got, ref, mag):
    """per-element relative error against the fp64 reference; NaN and +-Inf positions must be the reference's"""
    got, ref, mag = got.double().flatten(), ref.double().flatten(), mag.double().flatten()
    gn, rn = torch.isnan(got), torch.isnan(ref)
    assert torch.equal(gn, rn), (tag, "NaN positions differ", int((gn != rn).sum()))
    gi, ri = torch.isinf(got), torch.isinf(ref)
    assert torch.equal(gi, ri) and torch.equal(got[gi], ref[ri]), (tag, "Inf positions differ")
    fin = ~(rn | ri)
    e = float(((got - ref).abs()[fin] / (mag[fin] + 1e-300)).max()) if bool(fin.any()) else 0.0
    _WORST[tag] = max(_WORST.get(tag, 0.0), e)
    assert e <= TAU[tag], (tag, e, TAU[tag])
    return e


def _f32(b):
    return b.view(torch.float32)


def _f64(b):
    return b.view(F64)


def _inputs(n, s, c, seed, gamma=True, beta=True, res=True):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n * s * c, generator=gen, device=DEV) * 2 + 0.5
    dy = torch.randn(n * s * c, generator=gen, device=DEV)
    r = torch.randn(n * s * c, generator=gen, device=DEV) if res else None
    g = torch.rand(c, generator=gen, device=DEV) * 1.5 - 0.25 if gamma else None   # some weights negative, none near zero by design
    b = torch.randn(c, generator=gen, device=DEV) if beta else None
    return x, dy, r, g, b


def _groups(t, n, s, c, per_sample):
    """[G, M] fp64 view of a flat [n, s, c] tensor: one row per normalisation group (n * c of s, or c of n * s)"""
    t = t.double().view(n, s, c)
    return t.permute(0, 2, 1).reshape(n * c, s) if per_sample else t.permute(2, 0, 1).reshape(c, n * s)


def _bcast(stat, n, c, per_sample):
    """per-group statistic [G] -> broadcastable over [n, s, c]"""
    return stat.double().view(n, 1, c) if per_sample else stat.double().view(1, 1, c)


def _grad_rule(y, act):
    """torch's derivative of an in-place activation, from its output: ReLU y <= 0 -> 0 (else 1, NaN included), leaky ReLU y > 0 -> 1 else slope
    (fp32, as the kernels form it)"""
    if act == 0:
        return torch.ones_like(y)
    if act == 1:
        return torch.where(y <= 0, 0.0, 1.0)
    return torch.where(y > 0, 1.0, SLOPE)


def _act64(z, act):
    return z if act == 0 else F.relu(z) if act == 1 else F.leaky_relu(z, SLOPE)


def _stats_ref(x, n, s, c, per_sample):
    """fp64 mean, rstd, E[x^2], var and mean|x| per group"""
    xg = _groups(x, n, s, c, per_sample)
    mu, var = xg.mean(1), xg.var(1, unbiased=False)
    return dict(mean=mu, rstd=1 / torch.sqrt(var + EPS64), ex2=(xg * xg).mean(1), var=var, absmean=xg.abs().mean(1), m=xg.shape[1])


def _check_stats(st, mean, rstd, running=None, nbt=None, run0=None):
    """the kernel's mean / rstd (and running statistics, num_batches_tracked) against the fp64 statistics st"""
    _check("mean", mean, st["mean"], st["absmean"])
    _check("rstd", rstd, st["rstd"], st["rstd"] * (st["ex2"] + st["mean"] ** 2 + EPS64) / (st["var"] + EPS64))
    if running is not None:
        rm0, rv0 = (t.double() for t in run0)
        m = st["m"]
        _check("running_mean", running[0], (1 - MOM) * rm0 + MOM * st["mean"], (1 - MOM) * rm0.abs() + MOM * st["absmean"])
        _check("running_var", running[1], (1 - MOM) * rv0 + MOM * st["var"] * m / (m - 1),
               (1 - MOM) * rv0.abs() + MOM * (st["ex2"] + st["mean"] ** 2) * m / (m - 1))
    if nbt is not None:
        assert int(nbt) == 1


def _norm_ref(x, n, s, c, per_sample, gamma, beta, res, act, dy, y_kernel, batch_stats, mean=None, rstd=None):
    """fp64 y, and dx / dgamma / dbeta / dres by autograd of the same formula (F.batch_norm / F.instance_norm on [N, C, S], or the formula
    with the given mean / rstd as constants), with the activation's derivative taken from the kernel's output by torch's in-place rule
    (an fp32 pre-activation that rounds to the other side of 0 than the fp64 one changes nothing else).  Also the magnitudes (the same
    expressions on absolute values) of every output."""
    xl = x.double().view(n, s, c).requires_grad_(True)
    xn = xl.permute(0, 2, 1)
    w = (gamma.double() if gamma is not None else torch.ones(c, dtype=F64, device=DEV)).requires_grad_(True)
    b = beta.double() if beta is not None else None
    if batch_stats:
        st = _stats_ref(x, n, s, c, per_sample)
        mu, rs = st["mean"], st["rstd"]
        if per_sample:
            z = F.instance_norm(xn, weight=w, bias=b, eps=EPS64)
        else:
            z = F.batch_norm(xn, None, None, w, b, True, 0.0, EPS64)
    else:
        mu, rs = mean.double(), rstd.double()
        z = (xn - _bcast(mu, n, c, per_sample).permute(0, 2, 1)) * _bcast(rs, n, c, per_sample).permute(0, 2, 1) * w[:, None]
        if b is not None:
            z = z + b[:, None]
    z = z.permute(0, 2, 1)
    rl = res.double().view(n, s, c).requires_grad_(True) if res is not None else None
    if rl is not None:
        z = z + rl
    y_ref = _act64(z.detach(), act)
    g32 = dy.view(n, s, c) * _grad_rule(y_kernel.view(n, s, c), act)     # the kernels' fp32 g
    g = g32.double()
    grads = torch.autograd.grad(z, [xl, w] + ([rl] if rl is not None else []), grad_outputs=g)
    # magnitudes
    mu_e, rs_e = _bcast(mu, n, c, per_sample), _bcast(rs, n, c, per_sample)
    x64 = x.double().view(n, s, c)
    wa = w.detach().abs().view(1, 1, c)
    xh_mag = (x64.abs() + mu_e.abs()) * rs_e
    y_mag = wa * xh_mag + (b.abs().view(1, 1, c) if b is not None else 0) + (rl.detach().abs() if rl is not None else 0)
    ga = g.abs()
    if batch_stats:
        k1 = _bcast(_groups(ga, n, s, c, per_sample).mean(1), n, c, per_sample)
        k2 = _bcast(_groups(ga * xh_mag, n, s, c, per_sample).mean(1), n, c, per_sample)
        dx_mag = wa * rs_e * (ga + k1 + xh_mag * k2)
    else:
        dx_mag = wa * rs_e * ga
    return dict(y=y_ref, dx=grads[0], dgamma=grads[1], dbeta=g.sum((0, 1)), dres=g if rl is not None else None, g32=g32,
                y_mag=y_mag, dx_mag=dx_mag, dgamma_mag=(ga * xh_mag).sum((0, 1)), dbeta_mag=ga.sum((0, 1)), dres_mag=ga)


# ------------------------------------------------------------------------------------------------------------------------ ABI calls
def _stats(lib, x, n, s, c, per_sample, run0=None, eps=EPS):
    """mdt_norm_stats through guarded buffers -> (mean, rstd, [running_mean, running_var] or None, num_batches_tracked)"""
    groups = n * c if per_sample else c
    wsb = lib.mdt_norm_workspace_bytes(n, s, c, per_sample)
    assert wsb > 0
    running = [t.clone() for t in run0] if run0 is not None else None
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)

    def call(outs, ws):
        # the running buffers and the counter are updated in place: every run starts them from the same values
        if running is not None:
            running[0].copy_(run0[0])
            running[1].copy_(run0[1])
        nbt.zero_()
        rm, rv = (L.ptr(running[0]), L.ptr(running[1])) if running is not None else (None, None)
        return lib.mdt_norm_stats(L.ptr(x), n, s, c, per_sample, eps, MOM, outs[0], outs[1], rm, rv, L.ptr(nbt), ws, wsb, L.stream_ptr())

    mean_b, rstd_b = _run_guarded(call, [4 * groups, 4 * groups], wsb)
    return _f32(mean_b), _f32(rstd_b), running, nbt


def _apply(lib, x, mean, rstd, gamma, beta, res, n, s, c, per_sample, act):
    def call(outs, ws):
        return lib.mdt_norm_apply(L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(gamma), L.ptr(beta), L.ptr(res), n, s, c, per_sample, act, SLOPE, outs[0],
                                  L.stream_ptr())
    (y_b,) = _run_guarded(call, [4 * n * s * c], None)
    return _f32(y_b)


def _backward(lib, dy, y, x, mean, rstd, gamma, n, s, c, per_sample, act, batch_stats, want=(True, True, True)):
    """mdt_norm_backward through guarded buffers; want = (dgamma, dbeta, dresidual) set or NULL.  A call that needs no reduction (running
    statistics and no parameter gradient) gets a NULL workspace."""
    m = n * s * c
    reduce = batch_stats or want[0] or want[1]
    wsb = lib.mdt_norm_workspace_bytes(n, s, c, per_sample)

    def call(outs, ws):
        return lib.mdt_norm_backward(L.ptr(dy), L.ptr(y) if act else None, L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(gamma), n, s, c, per_sample,
                                     act, SLOPE, batch_stats, outs[0], outs[1], outs[2], outs[3], ws, wsb if reduce else 0, L.stream_ptr())
    outs = _run_guarded(call, [4 * m, 4 * c if want[0] else None, 4 * c if want[1] else None, 4 * m if want[2] else None], wsb if reduce else None)
    return [None if o is None else _f32(o) for o in outs]


def _pipeline(lib, case, seed, act, x=None, gamma=True, beta=True, res=True, dy=None):
    """stats -> apply -> backward (batch statistics, every output) of one case, each output checked against fp64; returns the outputs"""
    n, s, c, per_sample = case
    x0, dy0, r, g, b = _inputs(n, s, c, seed, gamma, beta, res)
    x = x0 if x is None else x
    dy = dy0 if dy is None else dy
    run0 = None if per_sample else [torch.randn(c, device=DEV) * 0.3, torch.rand(c, device=DEV) + 0.5]
    mean, rstd, running, nbt = _stats(lib, x, n, s, c, per_sample, run0)
    st = _stats_ref(x, n, s, c, per_sample)
    _check_stats(st, mean, rstd, running, nbt, run0)
    y = _apply(lib, x, mean, rstd, g, b, r, n, s, c, per_sample, act)
    ref = _norm_ref(x, n, s, c, per_sample, g, b, r, act, dy, y, 1)
    _check("y", y, ref["y"], ref["y_mag"])
    dx, dg, db, dr = _backward(lib, dy, y, x, mean, rstd, g, n, s, c, per_sample, act, 1, (True, True, r is not None))
    _check("dx", dx, ref["dx"], ref["dx_mag"])
    _check("dgamma", dg, ref["dgamma"], ref["dgamma_mag"])
    _check("dbeta", db, ref["dbeta"], ref["dbeta_mag"])
    if r is not None:
        assert torch.equal(dr.view(torch.int32), ref["g32"].reshape(-1).view(torch.int32)), "dresidual is not dy * act'(y) bit for bit"
        _check("dres", dr, ref["dres"], ref["dres_mag"])
    return dict(mean=mean, rstd=rstd, running=running, y=y, dx=dx, dgamma=dg, dbeta=db, dres=dr, gamma=g, beta=b, res=r, dy=dy)


# ------------------------------------------------------------------------------------------------------------------------ 1. split matrix
@pytest.mark.parametrize("case", M.SPLIT_CASES, ids=lambda c: "n%d-s%d-c%d-ps%d" % c)
def test_split_matrix(case):
    lib = L.load()
    _pipeline(lib, case, seed=sum(case), act=M.SPLIT_CASES.index(case) % 3)


# ------------------------------------------------------------------------------------------------------------------------ 2. backward arguments
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("with_gamma", [False, True])
@pytest.mark.parametrize("batch_stats", [0, 1])
@pytest.mark.parametrize("per_sample", [0, 1])
def test_backward_argument_matrix(per_sample, batch_stats, with_gamma, act):
    """every combination of dgamma / dbeta / dresidual set or NULL (dgamma NULL with dbeta set: a frozen weight); each set output fully
    written and right; running statistics and no parameter gradient run without a workspace"""
    lib = L.load()
    n, s, c = 3, 700, 20
    x, dy, r, g, b = _inputs(n, s, c, seed=31 + 4 * per_sample + 2 * batch_stats + with_gamma, gamma=with_gamma)
    mean, rstd, _, _ = _stats(lib, x, n, s, c, per_sample)
    if not batch_stats:   # constants unrelated to this batch
        mean, rstd = mean + 0.25, rstd * 0.75
    y = _apply(lib, x, mean, rstd, g, b, r, n, s, c, per_sample, act)
    ref = _norm_ref(x, n, s, c, per_sample, g, b, r, act, dy, y, batch_stats, mean, rstd)
    _check("y", y, ref["y"], ref["y_mag"])
    for want in [(dg, db, dr) for dg in (False, True) for db in (False, True) for dr in (False, True)]:
        dx, dgm, dbt, drs = _backward(lib, dy, y, x, mean, rstd, g, n, s, c, per_sample, act, batch_stats, want)
        _check("dx", dx, ref["dx"], ref["dx_mag"])
        if want[0]:
            _check("dgamma", dgm, ref["dgamma"], ref["dgamma_mag"])
        if want[1]:
            _check("dbeta", dbt, ref["dbeta"], ref["dbeta_mag"])
        if want[2]:
            assert torch.equal(drs.view(torch.int32), ref["g32"].reshape(-1).view(torch.int32))
            _check("dres", drs, ref["dres"], ref["dres_mag"])


# ------------------------------------------------------------------------------------------------------------------------ 3. eval statistics
@pytest.mark.parametrize("c", [1, 255, 257, 576])
def test_eval_stats(c):
    """mean = running_mean bit for bit; rstd = fp32(1 / sqrt(running_var + eps)) of the fp64 expression, bit for bit (IEEE sqrt and
    division), including running_var 0 and non-finite running statistics"""
    lib = L.load()
    gen = torch.Generator(device=DEV).manual_seed(c)
    rm = torch.randn(c, generator=gen, device=DEV) * 3
    rv = torch.rand(c, generator=gen, device=DEV) ** 4 * 10
    rv[0] = 0.0
    if c > 3:
        rv[1], rv[2], rm[3] = float("inf"), float("nan"), float("nan")
    mean_b, rstd_b = _run_guarded(lambda o, ws: lib.mdt_norm_eval_stats(L.ptr(rm), L.ptr(rv), c, EPS, o[0], o[1], L.stream_ptr()), [4 * c, 4 * c], None)
    mean, rstd = _f32(mean_b), _f32(rstd_b)
    assert torch.equal(mean.view(torch.int32), rm.view(torch.int32))
    want = (1.0 / np.sqrt(rv.cpu().numpy().astype(np.float64) + EPS64)).astype(np.float32)
    got = rstd.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok].view(np.int32), want[ok].view(np.int32))


# ------------------------------------------------------------------------------------------------------------------------ 4. synchronised path
SHARDS = [(0, None), (1, 1), (None, 1)]   # (local_first_row, n): the whole batch, one sample from row 1, the last sample


@pytest.mark.parametrize("case", M.SYNC_CASES, ids=lambda c: "n%d-s%d-c%d" % c)
def test_synchronised_entries(case):
    lib = L.load()
    n_total, s, c = case
    x, dy, r, g, b = _inputs(n_total, s, c, seed=n_total * 1000 + c)
    wsb_all = lib.mdt_norm_sample_workspace_bytes(n_total, s, c)
    xs = x.view(n_total, s * c)
    # per-sample sums of the whole batch (one rank holding every sample), guarded
    rows_b = _run_guarded(lambda o, ws: lib.mdt_norm_sample_sums(L.ptr(x), n_total, s, c, o[0], ws, wsb_all, L.stream_ptr()), [n_total * c * 16],
                          wsb_all)[0]
    rows = _f64(rows_b).view(n_total, c, 2)
    x64 = x.double().view(n_total, s, c)
    _check("sums_x", rows[..., 0], x64.sum(1), x64.abs().sum(1))
    _check("sums_x2", rows[..., 1], (x64 * x64).sum(1), (x64 * x64).sum(1))
    # statistics from the rows, guarded; running statistics and the counter in place
    run0 = [torch.randn(c, device=DEV) * 0.3, torch.rand(c, device=DEV) + 0.5]
    running = [t.clone() for t in run0]
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)

    def from_sums(o, ws):
        running[0].copy_(run0[0])
        running[1].copy_(run0[1])
        nbt.zero_()
        return lib.mdt_norm_stats_from_sums(L.ptr(rows), n_total, s, c, EPS, MOM, o[0], o[1], L.ptr(running[0]), L.ptr(running[1]), L.ptr(nbt),
                                            L.stream_ptr())
    mean, rstd = (_f32(t) for t in _run_guarded(from_sums, [4 * c, 4 * c], None))
    st = _stats_ref(x, n_total, s, c, 0)
    _check_stats(st, mean, rstd, running, nbt, run0)
    for k, act in enumerate((0, 1, 2)):
        first, n = SHARDS[k]
        first = n_total - 1 if first is None else first
        n = n_total if n is None else n
        lo, hi = first * s * c, (first + n) * s * c
        y = torch.empty_like(x)
        L.check(lib.mdt_norm_apply(L.ptr(x), L.ptr(mean), L.ptr(rstd), L.ptr(g), L.ptr(b), L.ptr(r), n_total, s, c, 0, act, SLOPE, L.ptr(y),
                                   L.stream_ptr()))
        # this shard's sums are the whole batch's rows of its samples, bit for bit
        wsb = lib.mdt_norm_sample_workspace_bytes(n, s, c)
        loc = _run_guarded(lambda o, ws: lib.mdt_norm_sample_sums(L.ptr(xs[first]), n, s, c, o[0], ws, wsb, L.stream_ptr()), [n * c * 16], wsb)[0]
        assert torch.equal(_f64(loc).view(n, c, 2), rows[first:first + n])
        # backward per-sample sums (sum g, sum g * xhat) against fp64 with the kernel's mean / rstd
        bl = _run_guarded(lambda o, ws: lib.mdt_norm_backward_sample_sums(L.ptr(dy[lo:]), L.ptr(y[lo:]) if act else None, L.ptr(xs[first]),
                                                                         L.ptr(mean), L.ptr(rstd), n, s, c, act, SLOPE, o[0], ws, wsb, L.stream_ptr()),
                          [n * c * 16], wsb)[0]
        bl = _f64(bl).view(n, c, 2)
        g32 = (dy * _grad_rule(y, act)).view(n_total, s, c)[first:first + n].double()
        xh = (x64[first:first + n] - mean.double()) * rstd.double()
        xh_mag = (x64[first:first + n].abs() + mean.double().abs()) * rstd.double()
        _check("bsums_g", bl[..., 0], g32.sum(1), g32.abs().sum(1))
        _check("bsums_gx", bl[..., 1], (g32 * xh).sum(1), (g32.abs() * xh_mag).sum(1))
        # the whole batch's backward rows (the exchange), then this shard's dx / dgamma / dbeta / dresidual
        grows = torch.empty(n_total, c, 2, dtype=F64, device=DEV)
        ws_all = torch.empty(wsb_all, dtype=torch.uint8, device=DEV)
        L.check(lib.mdt_norm_backward_sample_sums(L.ptr(dy), L.ptr(y) if act else None, L.ptr(x), L.ptr(mean), L.ptr(rstd), n_total, s, c, act, SLOPE,
                                                  L.ptr(grows), L.ptr(ws_all), wsb_all, L.stream_ptr()))
        assert torch.equal(grows[first:first + n], bl)
        outs = _run_guarded(lambda o, ws: lib.mdt_norm_backward_from_sums(
            L.ptr(dy[lo:]), L.ptr(y[lo:]) if act else None, L.ptr(xs[first]), L.ptr(mean), L.ptr(rstd), L.ptr(g), L.ptr(grows), n_total, first, n,
            s, c, act, SLOPE, o[0], o[1], o[2], o[3], ws, c * 16, L.stream_ptr()), [4 * n * s * c, 4 * c, 4 * c, 4 * n * s * c], c * 16)
        dx, dgm, dbt, drs = (_f32(o) for o in outs)
        ref = _norm_ref(x, n_total, s, c, 0, g, b, r, act, dy, y, 1)
        _check("y", y, ref["y"], ref["y_mag"])
        _check("dx", dx, ref["dx"][first:first + n], ref["dx_mag"][first:first + n])
        xh_ref = (x64 - st["mean"]) * st["rstd"]
        gl, xl, xm = ref["g32"][first:first + n].double(), xh_ref[first:first + n], ((x64.abs() + st["mean"].abs()) * st["rstd"])[first:first + n]
        _check("dgamma", dgm, (gl * xl).sum((0, 1)), (gl.abs() * xm).sum((0, 1)))
        _check("dbeta", dbt, gl.sum((0, 1)), gl.abs().sum((0, 1)))
        assert torch.equal(drs.view(torch.int32), ref["g32"][first:first + n].reshape(-1).view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------------ 5. activations
@pytest.mark.parametrize("count", [1, 4096 * 256 - 1, 4096 * 256 + 1, 3 * 4096 * 256 + 5])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_activation_grid_stride(count, act):
    """past one sweep of the 4096-block grid; the input holds exact zeros, NaN and +-Inf.  Forward bit for bit with F.relu / F.leaky_relu,
    backward bit for bit with dy * (torch's in-place rule on the output) and equal in value to torch's autograd of the in-place activation"""
    lib = L.load()
    gen = torch.Generator(device=DEV).manual_seed(count + act)
    x = torch.randn(count, generator=gen, device=DEV)
    x[::7] = 0.0
    if count > 100:
        x[1::97], x[2::89], x[3::83] = float("nan"), float("inf"), float("-inf")
        x[-1] = float("nan")
    (y_b,) = _run_guarded(lambda o, ws: lib.mdt_act_forward(L.ptr(x), count, act, SLOPE, o[0], L.stream_ptr()), [4 * count], None)
    y = _f32(y_b)
    want = x if act == 0 else F.relu(x) if act == 1 else F.leaky_relu(x, SLOPE)
    assert torch.equal(torch.isnan(y), torch.isnan(want))
    ok = ~torch.isnan(want)
    assert torch.equal(y[ok].view(torch.int32), want[ok].view(torch.int32))
    dy = torch.randn(count, generator=gen, device=DEV)
    (dx_b,) = _run_guarded(lambda o, ws: lib.mdt_act_backward(L.ptr(dy), L.ptr(y) if act else None, count, act, SLOPE, o[0], L.stream_ptr()),
                           [4 * count], None)
    dx = _f32(dx_b)
    assert torch.equal(dx.view(torch.int32), (dy * _grad_rule(y, act)).view(torch.int32))
    if act:
        xl = x.clone().requires_grad_(True)
        t = xl * 1.0
        out = F.relu(t, inplace=True) if act == 1 else F.leaky_relu(t, SLOPE, inplace=True)
        (gx,) = torch.autograd.grad(out, xl, dy)
        assert torch.equal(dx, gx)


# ------------------------------------------------------------------------------------------------------------------------ 6. values at the edges
def _poison_case(per_sample):
    return (3, 500, 20, per_sample)


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("value", ["nan", "inf"])
@pytest.mark.parametrize("per_sample", [0, 1])
def test_non_finite_value_poisons_exactly_its_group(per_sample, value, act):
    """one NaN or +Inf at (sample 1, row 37, channel 5): every output of that group (instance norm: (1, 5); batch norm: channel 5) is
    what fp64 torch gives (NaN: also the running statistics), and every other group is unaffected"""
    lib = L.load()
    case = _poison_case(per_sample)
    n, s, c, _ = case
    x, _, _, _, _ = _inputs(n, s, c, seed=77 + per_sample)
    x = x.clone()
    x.view(n, s, c)[1, 37, 5] = float(value)
    out = _pipeline(lib, case, seed=77 + per_sample, act=act, x=x)
    y = out["y"].view(n, s, c)
    grp = torch.zeros(n, s, c, dtype=torch.bool, device=DEV)
    if per_sample:
        grp[1, :, 5] = True
    else:
        grp[:, :, 5] = True
    assert bool(torch.isnan(y[grp]).all()) and bool(torch.isfinite(y[~grp]).all())
    assert bool(torch.isnan(out["dx"].view(n, s, c)[grp]).all()) and bool(torch.isfinite(out["dx"].view(n, s, c)[~grp]).all())
    if not per_sample:
        rm, rv = out["running"]
        assert bool(torch.isnan(rv[5])) and bool(torch.isfinite(rv[torch.arange(c, device=DEV) != 5]).all())
        assert (bool(torch.isnan(rm[5])) if value == "nan" else float(rm[5]) == float("inf"))


@pytest.mark.parametrize("per_sample", [0, 1])
def test_constant_group(per_sample):
    """a constant group has variance 0: rstd = fp32(1 / sqrt(eps)) and y = beta, bit for bit"""
    lib = L.load()
    case = (3, 500, 20, per_sample)
    n, s, c, _ = case
    x, _, _, _, _ = _inputs(n, s, c, seed=5)
    x = x.clone()
    xv = x.view(n, s, c)
    if per_sample:
        xv[2, :, 7] = 0.75
    else:
        xv[:, :, 7] = 0.75
    out = _pipeline(lib, case, seed=5, act=0, x=x, res=False)
    grp = 2 * c + 7 if per_sample else 7
    assert float(out["rstd"][grp]) == float(np.float32(1.0 / np.sqrt(EPS64)))
    yg = out["y"].view(n, s, c)[2, :, 7] if per_sample else out["y"].view(n, s, c)[:, :, 7]
    assert bool((yg == out["beta"][7]).all())


@pytest.mark.parametrize("per_sample", [0, 1])
def test_offset_data(per_sample):
    """mean 1e4, spread 1e-3 (a few fp32 ulps at 1e4): E[x^2] - mean^2 cancels to within rounding and may come out negative; the clamp
    keeps every output finite"""
    lib = L.load()
    case = (3, 900, 20, per_sample)
    n, s, c, _ = case
    gen = torch.Generator(device=DEV).manual_seed(12)
    x = 1e4 + 1e-3 * torch.randn(n * s * c, generator=gen, device=DEV)
    out = _pipeline(lib, case, seed=12, act=2, x=x)
    for k in ("mean", "rstd", "y", "dx", "dgamma", "dbeta"):
        assert bool(torch.isfinite(out[k]).all()), k


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("per_sample", [0, 1])
def test_pre_activation_exactly_zero(per_sample, act):
    """outputs exactly at 0 take torch's in-place derivative there (ReLU 0, leaky ReLU the slope): (a) gamma = beta = residual = 0, against
    fp64 torch autograd through F.relu_ / F.leaky_relu_; (b) gamma = 1, beta = 0 and residual = -xhat of the kernel's own statistics: the
    normalised value is rounded once before the residual add, so the sum is exactly 0"""
    lib = L.load()
    n, s, c = 2, 600, 9
    x, dy, _, _, _ = _inputs(n, s, c, seed=40 + act)
    mean, rstd, _, _ = _stats(lib, x, n, s, c, per_sample)
    zero_c, zero_x = torch.zeros(c, device=DEV), torch.zeros_like(x)
    # (a)
    y = _apply(lib, x, mean, rstd, zero_c, zero_c, zero_x, n, s, c, per_sample, act)
    assert bool((y == 0).all())
    dx, dg, db, dr = _backward(lib, dy, y, x, mean, rstd, zero_c, n, s, c, per_sample, act, 1)
    xl = x.double().view(n, s, c).requires_grad_(True)
    w, b = torch.zeros(c, dtype=F64, device=DEV, requires_grad=True), torch.zeros(c, dtype=F64, device=DEV, requires_grad=True)
    rl = torch.zeros(n, s, c, dtype=F64, device=DEV, requires_grad=True)
    xn = xl.permute(0, 2, 1)
    z = (F.instance_norm(xn, weight=w, bias=b, eps=EPS64) if per_sample else F.batch_norm(xn, None, None, w, b, True, 0.0, EPS64)).permute(0, 2, 1) + rl
    z = F.relu(z, inplace=True) if act == 1 else F.leaky_relu(z, SLOPE, inplace=True)
    gx, gw, gb, gr = torch.autograd.grad(z, [xl, w, b, rl], dy.double().view(n, s, c))
    assert bool((gr == 0).all()) if act == 1 else bool((gr == SLOPE * dy.double().view(n, s, c)).all())
    _check("dres", dr, gr, gr.abs())
    _check("dbeta", db, gb, gr.abs().sum((0, 1)))
    ref = _norm_ref(x, n, s, c, per_sample, zero_c, zero_c, zero_x, act, dy, y, 1)
    _check("dgamma", dg, gw, ref["dgamma_mag"])
    assert bool((dx == 0).all()) and bool((gx == 0).all())
    # (b)
    grp = _bcast(torch.arange(mean.numel(), device=DEV), n, c, per_sample).long().expand(n, s, c).reshape(-1)
    res = -((x - mean[grp]) * rstd[grp])
    one_c = torch.ones(c, device=DEV)
    y = _apply(lib, x, mean, rstd, one_c, zero_c, res, n, s, c, per_sample, act)
    assert bool((y == 0).all())
    dx, dg, db, dr = _backward(lib, dy, y, x, mean, rstd, one_c, n, s, c, per_sample, act, 1)
    assert torch.equal(dr, dy * (0.0 if act == 1 else SLOPE))
    ref = _norm_ref(x, n, s, c, per_sample, one_c, zero_c, res, act, dy, y, 1)
    _check("dx", dx, ref["dx"], ref["dx_mag"])
    _check("dgamma", dg, ref["dgamma"], ref["dgamma_mag"])
    _check("dbeta", db, ref["dbeta"], ref["dbeta_mag"])


# ------------------------------------------------------------------------------------------------------------------------ 7. the metric
def test_metric_catches_a_planted_split_error():
    """the 33-chunk batch-norm case against references with a split slip planted in them: the 33rd row block (the one lane 0 of the
    finalising warp folds second) left out of every channel's sums, or every block-33 partial handed to the next channel.  Each must fail the
    metric of mean, rstd, dgamma and dbeta by far more than its bound."""
    lib = L.load()
    case = (3, 176, 256, 0)
    n, s, c, _ = case
    g = M.make_geo(*case)
    assert g.chunks == 33
    out = _pipeline(lib, case, seed=3, act=2)
    x = _inputs(n, s, c, seed=3)[0]
    lo, hi = 32 * g.rows, min(33 * g.rows, g.R)
    xg = _groups(x, n, s, c, 0)
    gg = _groups(out["dres"], n, s, c, 0)            # g = dy * act'(y)
    xh = (xg - xg.mean(1, keepdim=True)) / torch.sqrt(xg.var(1, unbiased=False, keepdim=True) + EPS64)
    terms = {"x": xg, "x2": xg * xg, "g": gg, "gx": gg * xh}
    full = {k: v.sum(1) for k, v in terms.items()}
    block = {k: v[:, lo:hi].sum(1) for k, v in terms.items()}
    plants = {"dropped": {k: full[k] - block[k] for k in terms},
              "neighbour": {k: full[k] - block[k] + torch.roll(block[k], 1) for k in terms}}
    absx = xg.abs().mean(1)
    for name, p in plants.items():
        mu = p["x"] / g.R
        var = p["x2"] / g.R - mu * mu
        rs = 1 / torch.sqrt(var.clamp_min(0) + EPS64)
        es = {"mean": (out["mean"].double() - mu).abs() / absx,
              "rstd": (out["rstd"].double() - rs).abs() / (rs * (p["x2"] / g.R + mu * mu + EPS64) / (var.clamp_min(0) + EPS64)),
              "dgamma": (out["dgamma"].double() - p["gx"]).abs() / (gg.abs() * (xg.abs() + xg.mean(1, keepdim=True).abs()) /
                                                                    torch.sqrt(xg.var(1, unbiased=False, keepdim=True) + EPS64)).sum(1),
              "dbeta": (out["dbeta"].double() - p["g"]).abs() / gg.abs().sum(1)}
        for k, e in es.items():
            e = float(e.max())
            print("planted %s: e(%s) = %.3g (bound %.3g)" % (name, k, e, TAU[k]))
            assert e >= 3 * TAU[k], (name, k, e, TAU[k])
