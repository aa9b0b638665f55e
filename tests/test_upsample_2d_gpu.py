"""Bilinear x2 (2D) and (2,2,1) trilinear (3D) up-sampling at any channel count on the library (csrc/resample.cu:
mdt_upsample_linear2x_forward / _backward), and bit-reproducible 2D training of every model that runs the full-resolution decoder (GPU).

  * op: C in {1, 2, 3, 4, 6, 36, 192}, extents 1-3 and odd sizes, 2D maps (w = 1) and 3D maps (w > 1), through poisoned exact-size buffers
    (tests/_guarded.py): forward against fp64 F.interpolate, backward against its fp64 adjoint, within tests/test_ops_edges_gpu.py's "up221"
    bound; every guarded offset gives the same bits;
  * path independence: the V = 4, 2 and 1 channel accesses give the same bits, and at C % 4 == 0 the new entries equal mdt_upsample221_*;
  * non-finite inputs: NaN and Inf land where fp64 torch puts them.  torch's kernel reads input 1 with weight 0 for output 0 of a scaled axis
    (and its backward adds 0 x gy[0] into gx[1]), so a non-finite there makes torch's value NaN where the exact value is finite; those
    positions are checked against the exact value instead;
  * models: two 2D train steps from the same weights and batch give bit-identical losses, parameter gradients (fpn P1 / P0 included) and
    buffers, and two runs of three Adam steps bit-identical parameters, for Retina U-Net (lidc; instance norm + leaky ReLU; batch norm; the
    two-channel PET-CT config), UFRCNN+, the Detection U-Net and RetinaNet;
  * a 2D train step of each full-resolution model launches no up-sampling kernel outside the library."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _guarded import DEV, _run_guarded
from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import backbone as B
from test_ops_edges_gpu import CL3, MDT_EINVAL, _as, _check, _misaligned, _ptr, _sp, _vec

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

# (d, h, w): the 2D maps are [n, c, d, h] viewed with w = 1
SHAPES_2D = [(d, h, 1) for d in (1, 2, 3) for h in (1, 2, 3)] + [(5, 7, 1), (9, 4, 1)]
SHAPES_3D = [(1, 3, 2), (3, 2, 5), (4, 5, 3)]


def _map(n, C, sp, seed):
    torch.manual_seed(seed)
    return torch.randn((n, C) + sp, device=DEV).contiguous(memory_format=CL3)


def _up64(t):
    """fp64 F.interpolate of a [n, C, d, h, w] map: bilinear x2 on [n, C, d, h] when w == 1, else trilinear (2,2,1)"""
    if t.shape[-1] == 1:
        return F.interpolate(t[..., 0], scale_factor=2, mode="bilinear", align_corners=False).unsqueeze(-1)
    return F.interpolate(t, scale_factor=(2, 2, 1), mode="trilinear", align_corners=False)


def _fwd(x, offsets=None, entry="mdt_upsample_linear2x_forward"):
    n, C, d, h, w = x.shape
    call = lambda o, ws: getattr(L.load(), entry)(L.ptr(x), o[0], n, d, h, w, C, _sp())   # noqa: E731
    kw = {} if offsets is None else dict(offsets=offsets)
    y_b = _run_guarded(call, [4 * 4 * x.numel()], None, **kw)[0]
    return _as(y_b, torch.float32, n, 2 * d, 2 * h, w, C).permute(0, 4, 1, 2, 3)


def _bwd(gy, offsets=None, entry="mdt_upsample_linear2x_backward"):
    n, C, od, oh, w = gy.shape
    call = lambda o, ws: getattr(L.load(), entry)(L.ptr(gy), o[0], n, od // 2, oh // 2, w, C, _sp())   # noqa: E731
    kw = {} if offsets is None else dict(offsets=offsets)
    gx_b = _run_guarded(call, [gy.numel()], None, **kw)[0]
    return _as(gx_b, torch.float32, n, od // 2, oh // 2, w, C).permute(0, 4, 1, 2, 3)


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ================================================================================================================================ op
@pytest.mark.parametrize("C", [1, 2, 3, 4, 6, 36, 192])
def test_forward_and_adjoint_vs_fp64(C):
    for k, sp in enumerate(SHAPES_2D + SHAPES_3D):
        x = _map(2, C, sp, seed=C * 100 + k)
        y = _fwd(x)
        x64 = x.double().requires_grad_(True)
        ref = _up64(x64)
        _check("up221", y, ref.detach(), _up64(x.double().abs()))
        gy = torch.randn(ref.shape, device=DEV).contiguous(memory_format=CL3)
        gx = _bwd(gy)
        ref.backward(gy.double())
        xa = x.double().requires_grad_(True)
        _up64(xa).backward(gy.double().abs())
        _check("up221", gx, x64.grad, xa.grad)


def test_argument_errors():
    lib = L.load()
    x = torch.randn(1, 3, 2, 2, 1, device=DEV).contiguous(memory_format=CL3)
    y = torch.empty(4 * x.numel() + 4, device=DEV)
    for fn in (lib.mdt_upsample_linear2x_forward, lib.mdt_upsample_linear2x_backward):
        assert fn(None, L.ptr(y), 1, 2, 2, 1, 3, _sp()) == MDT_EINVAL
        assert fn(L.ptr(x), None, 1, 2, 2, 1, 3, _sp()) == MDT_EINVAL
        for bad in ((0, 2, 2, 1, 3), (1, 0, 2, 1, 3), (1, 2, 0, 1, 3), (1, 2, 2, 0, 3), (1, 2, 2, 1, 0)):
            assert fn(L.ptr(x), L.ptr(y), *bad, _sp()) == MDT_EINVAL
        assert fn(_ptr(x, 2), L.ptr(y), 1, 2, 2, 1, 3, _sp()) == MDT_EINVAL        # not 4-byte aligned
        assert fn(L.ptr(x), _ptr(y, 1), 1, 2, 2, 1, 3, _sp()) == MDT_EINVAL


@pytest.mark.parametrize("C", [4, 36, 192, 2, 6, 3])
@pytest.mark.parametrize("sp", [(5, 7, 1), (3, 2, 5)], ids=["2d", "3d"])
def test_vector_widths_give_the_same_bits(C, sp):
    """input and output both at 0, 8 and 4 bytes past a 16-byte boundary select V = 4, 2, 1 (as C allows): same bits forward and backward;
    at C % 4 == 0 the float4-only mdt_upsample221_* give the same bits too"""
    x0 = _map(2, C, sp, seed=C)
    gy0 = _map(2, C, (2 * sp[0], 2 * sp[1], sp[2]), seed=C + 1)
    ys, gxs = {}, {}
    for floats in (0, 2, 1):
        want = {0: 4 if C % 4 == 0 else 2 if C % 2 == 0 else 1, 2: 2 if C % 2 == 0 else 1, 1: 1}[floats]
        x, gy, off = _misaligned(x0, floats), _misaligned(gy0, floats), 4 * floats
        assert _vec(C, x.data_ptr(), off) == want and _vec(C, gy.data_ptr(), off) == want
        ys[floats] = _fwd(x, offsets=(off, 256 + off))
        gxs[floats] = _bwd(gy, offsets=(off, 256 + off))
    for f in (2, 1):
        assert _bits(ys[f], ys[0]) and _bits(gxs[f], gxs[0]), f
    if C % 4 == 0:
        assert _bits(_fwd(x0, entry="mdt_upsample221_forward"), ys[0])
        assert _bits(_bwd(gy0, entry="mdt_upsample221_backward"), gxs[0])


def _same_nonfinite(got, ref):
    """NaN where ref is NaN, the same infinity where ref is infinite, and finite elsewhere"""
    assert torch.equal(torch.isnan(got), torch.isnan(ref.float()))
    inf = torch.isinf(ref)
    assert torch.equal(torch.isinf(got), inf) and torch.equal(got[inf].double(), ref[inf])


@pytest.mark.parametrize("C", [3, 36])
def test_non_finite_inputs(C):
    """2D maps: NaN / +Inf / -Inf at random positions of x (forward) and gy (backward) land where fp64 torch puts them; the finite elements
    stay within the "up221" bound of the same computation with the non-finite inputs replaced by 0"""
    sp = (6, 5, 1)
    rs = np.random.RandomState(C)
    x = _map(2, C, sp, seed=7)
    gy = _map(2, C, (12, 10, 1), seed=8)
    vals = [float("nan"), float("inf"), -float("inf")]
    # torch's zero-weight reads (input 1 in the forward, output 0 in the backward along a scaled axis) are left out here, see below
    for t, skip in ((x, 1), (gy, 0)):
        for k in range(6):
            i, j = [int(rs.choice([a for a in range(n) if a != skip])) for n in t.shape[2:4]]
            t[int(rs.randint(2)), int(rs.randint(C)), i, j, 0] = vals[k % 3]
    y, gx = _fwd(x), _bwd(gy)
    ref = _up64(x.double())
    _same_nonfinite(y, ref)
    x64 = x.double().requires_grad_(True)
    _up64(x64).backward(gy.double())
    _same_nonfinite(gx, x64.grad)
    fin = lambda t: torch.where(torch.isfinite(t), t, torch.zeros_like(t))   # noqa: E731
    ok = torch.isfinite(ref)
    _check("up221", y[ok], _up64(fin(x).double())[ok], _up64(fin(x).double().abs())[ok])
    x0 = fin(x).double().requires_grad_(True)
    xa = fin(x).double().requires_grad_(True)
    _up64(x0).backward(fin(gy).double())
    _up64(xa).backward(fin(gy).double().abs())
    okg = torch.isfinite(x64.grad)
    _check("up221", gx[okg], x0.grad[okg], xa.grad[okg])


def test_non_finite_at_torchs_zero_weight_taps():
    """x[1] = Inf along h: torch gives NaN at output 0 (0 x Inf), the exact value x[0] is finite and the library returns it.  gy[0] = Inf along
    h: torch gives NaN at gx[1]; the library puts +Inf at gx[0] only"""
    C = 4
    x = _map(1, C, (4, 3, 1), seed=3)
    x[0, 1, 1, 2, 0] = float("inf")
    y = _fwd(x)
    assert bool(torch.isnan(_up64(x.double())[0, 1, 0]).any())
    x0 = x.clone()
    x0[0, 1, 1, 2, 0] = 0.0
    _check("up221", y[:, :, 0], _up64(x0.double())[:, :, 0], _up64(x0.double().abs())[:, :, 0])
    gy = _map(1, C, (8, 6, 1), seed=4)
    gy[0, 2, 0, 3, 0] = float("inf")
    gx = _bwd(gy)
    x64 = x.double().requires_grad_(True)
    _up64(x64).backward(gy.double())
    assert bool(torch.isnan(x64.grad[0, 2, 1]).any())
    assert bool(torch.isposinf(gx[0, 2, 0, 1:3, 0]).all()) and int(torch.isinf(gx).sum()) == 2 and not bool(torch.isnan(gx).any())


# ============================================================================================================================ models
PETCT = 'pet_ct_tnm_classification'


def _cf_retina(model="retina_unet", exp="lidc_exp", **over):
    from medicaldetectiontoolkit_b200.configs import make_cf
    cf = make_cf(model, 2, (128, 128), exp=exp, batch_size=2)
    for k, v in over.items():
        setattr(cf, k, v)
    return cf


def _retina(model="retina_unet", exp="lidc_exp", **over):
    from medicaldetectiontoolkit_b200 import retina_net, retina_unet
    from medicaldetectiontoolkit_b200.configs import synthetic_batch
    cf = _cf_retina(model, exp, **over)
    mod = retina_unet if model == "retina_unet" else retina_net
    torch.manual_seed(0)
    net = mod.net(cf, None).to(DEV)
    batch = synthetic_batch(cf, 2, seed=1)
    if exp == PETCT:                                   # the experiment's single foreground class
        batch['roi_labels'] = [np.ones_like(lab) for lab in batch['roi_labels']]
    return net, batch


def _det_unet():
    from medicaldetectiontoolkit_b200 import detection_unet
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    cf = make_cf('detection_unet', 2, (128, 128))
    torch.manual_seed(0)
    return detection_unet.net(cf).to(DEV), synthetic_batch(cf, 2, seed=3)


def _ufrcnn_2d():
    sys.path.insert(0, GOLD)
    import make_ufrcnn_golden as G
    from medicaldetectiontoolkit_b200 import ufrcnn as UF
    cf = G.case_cf("2d")
    g = np.load(os.path.join(GOLD, "ufrcnn_model_2d.npz"))
    return G.weights_(UF.net(cf)).to(DEV), G.batch_from_golden(cf, g, "2d")


MODELS = {
    "retina_unet_lidc": lambda: _retina(),
    "retina_unet_in_leaky": lambda: _retina(norm="instance_norm", relu="leaky_relu"),
    "retina_unet_bn": lambda: _retina(norm="batch_norm"),
    "retina_unet_petct": lambda: _retina(exp=PETCT),
    "ufrcnn_2d": _ufrcnn_2d,
    "det_unet_2d": _det_unet,
    "retina_net_2d": lambda: _retina("retina_net"),
}
FULL_RES = ["retina_unet_lidc", "ufrcnn_2d", "det_unet_2d"]


def _step(net, batch):
    torch.manual_seed(1)
    np.random.seed(1)
    net.zero_grad(set_to_none=True)
    res = net.train_forward(batch)
    res['torch_loss'].backward()
    return res


@pytest.mark.parametrize("case", list(MODELS))
def test_2d_train_steps_are_bit_identical(case, monkeypatch):
    from medicaldetectiontoolkit_b200 import model_utils as mutils
    monkeypatch.setattr(mutils, "SAMPLING", "random")
    net, batch = MODELS[case]()
    state = copy.deepcopy(net.state_dict())

    def run():
        net.load_state_dict(state)
        loss = float(_step(net, batch)['torch_loss'])
        return loss, {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}, \
            {k: b.clone() for k, b in net.named_buffers()}
    l1, g1, b1 = run()
    l2, g2, b2 = run()
    assert np.isfinite(l1) and l1 == l2 and sorted(g1) == sorted(g2)
    assert [k for k in g1 if not torch.equal(g1[k], g2[k])] == []
    assert [k for k in b1 if not torch.equal(b1[k], b2[k])] == []
    if case != "retina_net_2d":                        # the decoder's P1 / P0 path receives the up-sampling backward
        for name in ("P1_conv1.weight", "P0_conv1.weight"):
            k = next(k for k in g1 if k.lower().endswith("fpn." + name.lower()))
            assert float(g1[k].abs().sum()) > 0, k

    def train3():
        net.load_state_dict(state)
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        for _ in range(3):
            _step(net, batch)
            opt.step()
        return {k: p.detach().clone() for k, p in net.named_parameters()}
    p1, p2 = train3(), train3()
    assert [k for k in p1 if not torch.equal(p1[k], p2[k])] == []


@pytest.mark.parametrize("case", FULL_RES)
def test_no_torch_upsampling_kernel_in_a_2d_step(case, monkeypatch):
    from medicaldetectiontoolkit_b200 import model_utils as mutils
    monkeypatch.setattr(mutils, "SAMPLING", "random")
    net, batch = MODELS[case]()
    _step(net, batch)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _step(net, batch)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert not sorted(k for k in names if "mdt::" not in k and "upsample" in k.lower())
    assert any("mdt::upsample221_fwd_kernel" in k for k in names) and any("mdt::upsample221_bwd_kernel" in k for k in names)


def test_interpolate_module_paths():
    """Interpolate sends 4-D bilinear x2 and 5-D (2,2,1) trilinear at any C to the library, with torch's values to the fp32 rounding of
    the fp64 reference; misaligned views are copied; CPU maps keep F.interpolate"""
    for shape, kw in (((2, 6, 5, 7), dict(scale_factor=2, mode='bilinear')), ((2, 6, 5, 7, 3), dict(scale_factor=(2, 2, 1), mode='trilinear')),
                      ((2, 36, 5, 7), dict(scale_factor=(2, 2), mode='bilinear'))):
        torch.manual_seed(len(shape))
        mf = torch.channels_last if len(shape) == 4 else CL3
        x = _misaligned(torch.randn(shape, device=DEV).contiguous(memory_format=mf))
        assert x.is_contiguous(memory_format=mf) and x.data_ptr() % 16 == 4
        xg = x.detach().requires_grad_(True)
        y = B.Interpolate(**kw)(xg)
        assert y.is_contiguous(memory_format=mf)
        x64 = x.detach().double().requires_grad_(True)
        ref = F.interpolate(x64, align_corners=False, **kw)
        assert torch.allclose(y.double(), ref, rtol=1e-6, atol=1e-6)
        g = torch.randn(y.shape, device=DEV)
        gx, = torch.autograd.grad(y, xg, g)
        ref.backward(g.double())
        assert torch.allclose(gx.double(), x64.grad, rtol=1e-6, atol=1e-5)
        gx2, = torch.autograd.grad(B.Interpolate(**kw)(xg), xg, g)
        assert torch.equal(gx, gx2)
        xc = x.detach().cpu()
        assert torch.equal(B.Interpolate(**kw)(xc), F.interpolate(xc, align_corners=False, **kw))
