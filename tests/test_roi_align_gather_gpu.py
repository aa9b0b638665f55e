"""The RoIAlign backward is a gather with a fixed summation order (csrc/roi_align.cu: roi_bwd_gather), so its result is a specified function of
its inputs and Mask R-CNN / UFRCNN+ training is bit-reproducible (GPU).

  * specified result: every entry point, on every layout of tests/test_ops_edges_gpu.py::ROI_CASES and on a 4-level pyramid in 2D and 3D,
    through poisoned exact-size buffers with zero_init 1 and 0, equals the host restatement tests/roi_gather_model.c bit for bit (and stays
    within the fp64 adjoint's tau);
  * path independence: the channels-last vector path, the strided scalar path (misaligned, NCDHW) and the pyramid give the same bits;
  * the cases the float atomics used to hide: hundreds of identical boxes, more overlapping RoIs than one shared-memory chunk, boxes clamped at
    the border, inverted boxes and crop extent 1, bad box_ind next to good ones (with NaN rows), Inf gradients behind zero-weight corners;
  * whole models: two Mask R-CNN (3D small and cfg3, 2D) and UFRCNN+ (3D small) train steps give bit-identical parameter gradients, and
    three Adam steps bit-identical parameters.  UFRCNN+ in 2D is not covered: its full-resolution decoder up-samples P2 -> P1 -> P0 with
    torch's bilinear F.interpolate, whose CUDA backward adds with atomics, so fpn.P1_conv1 and the layers below it still differ from run to
    run (every gradient the RoIAlign backward feeds agrees)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import _roi_gather_model as M
from _guarded import DEV, OFFSETS, _Guarded, _run_guarded
from medicaldetectiontoolkit_b200 import _lib as L
from test_ops_edges_gpu import (CL3, ROI_CASES, TAU, _cl_strides, _crop_nbytes, _err, _i32, _roi_boxes, _roi_case, _roi_path,
                                _roi_ref_bwd, _sp, _strides5)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _bwd_call(g, gs5, boxes_t, ind_t, crop, is5, shape, numel, zero_init):
    lib, dim, n = L.load(), len(crop), boxes_t.shape[0]
    C, sp = shape[1], shape[2:]
    if dim == 3:
        return lambda o, ws: lib.mdt_crop_and_resize_3d_backward(L.ptr(g), L.i64arr(gs5), L.ptr(boxes_t), L.ptr(ind_t), n, shape[0], *sp, *crop, C, o[0],
                                                                 L.i64arr(is5), zero_init, numel, _sp())
    return lambda o, ws: lib.mdt_crop_and_resize_2d_backward(L.ptr(g), L.i64arr(gs5[:4]), L.ptr(boxes_t), L.ptr(ind_t), n, shape[0], *sp, *crop, C, o[0],
                                                             L.i64arr(is5[:4]), zero_init, numel, _sp())


def _run_prior(call, prior_bytes, offsets=OFFSETS):
    """call(out_ptrs, None) once per base offset with each output an exact-size guarded view that starts as `prior_bytes` (zero_init = 0);
    guards intact, every run the same bits; returns the first run's outputs"""
    runs = []
    for off in offsets:
        outs = [_Guarded(p.numel(), off, 0) for p in prior_bytes]
        for o, p in zip(outs, prior_bytes):
            o.data().copy_(p)
        L.check(call([o.ptr() for o in outs], None))
        torch.cuda.synchronize()
        for o in outs:
            o.check_guards()
        runs.append([o.data().clone() for o in outs])
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))
    return runs[0]


def _f32(b):
    return b.view(torch.float32).cpu().numpy()


def _model(g_flat, gs5, boxes, ind, prior, is5, shape, crop, zero_init, **kw):
    return M.gather_backward(g_flat, gs5, boxes, ind, prior.copy(), is5, shape, crop, zero_init, **kw)


def _same_bits(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    diff = got.view(np.uint32) != want.view(np.uint32)
    assert not diff.any(), "%d of %d elements differ, first at %d: %r vs %r" % (diff.sum(), diff.size, np.flatnonzero(diff)[0],
                                                                                got.ravel()[diff.ravel()][0], want.ravel()[diff.ravel()][0])


def _check_entry(call, g_flat, gs5, boxes, ind, shape, is5, crop, nbytes, offs, model_kw=None, adjoint=None):
    """zero_init 1 through poisoned buffers and zero_init 0 over a finite prior: both equal the restatement bit for bit"""
    model_kw = model_kw or {}
    nel = nbytes // 4
    out = _run_guarded(lambda o, ws: call(1)(o, ws), [nbytes], None, offsets=offs)[0]
    got = _f32(out)
    _same_bits(got, _model(g_flat, gs5, boxes, ind, np.zeros(nel, np.float32), is5, shape, crop, 1, **model_kw))
    if adjoint is not None:
        gx = torch.as_strided(out.view(torch.float32), shape, is5[:len(shape)])
        e = _err(gx, *adjoint)
        assert e <= TAU["roi-bwd"], e
    prior = torch.randn(nel, generator=torch.Generator().manual_seed(nel)).float()
    out0 = _run_prior(lambda o, ws: call(0)(o, ws), [prior.view(torch.uint8).to(DEV)], offsets=offs)[0]
    _same_bits(_f32(out0), _model(g_flat, gs5, boxes, ind, prior.numpy(), is5, shape, crop, 0, **model_kw))
    return got


def _grads(cshape, os5, nb, seed=3):
    torch.manual_seed(seed)
    base = torch.randn(nb // 4, device=DEV)
    return base, torch.as_strided(base, cshape, os5[:len(cshape)])


@pytest.mark.parametrize("case", ROI_CASES, ids=[c[0] for c in ROI_CASES])
def test_backward_is_the_specified_sum(case):
    img, shape, cshape, os5, boxes, ind, path = _roi_case(case)
    dim, crop = case[1], case[5]
    is5 = _strides5(img.stride())
    nb = _crop_nbytes(cshape, os5[:dim + 2])
    base, g = _grads(cshape, os5, nb)
    boxes_t, ind_t = torch.from_numpy(boxes).to(DEV), torch.from_numpy(ind).to(DEV)
    numel = int(np.prod(shape))
    offs = (4, 260, 772) if case[6] == "cl_mis" else (0, 256, 768)
    assert _roi_path(case[3], crop, is5, os5, offs[0], g.data_ptr(), case[4]) == path
    _check_entry(lambda z: _bwd_call(g, os5, boxes_t, ind_t, crop, is5, shape, numel, z), base.cpu().numpy(), os5, boxes, ind, shape, is5, crop,
                 numel * 4, offs, adjoint=_roi_ref_bwd(g, boxes, ind, crop, shape))


def _pyr_setup(dim, C=36, n=40, seed=5):
    crop = (7, 7, 3) if dim == 3 else (7, 7)
    sps = [(32, 32, 16), (16, 16, 8), (8, 8, 4), (4, 4, 2)] if dim == 3 else [(48, 40), (24, 20), (12, 10), (6, 5)]
    mf = CL3 if dim == 3 else torch.channels_last
    boxes, ind = _roi_boxes(n, dim, 2, seed=seed)
    level = np.random.RandomState(seed).randint(-1, 5, size=n).astype(np.int32)      # -1 and 4 are clamped to levels 0 and 3
    torch.manual_seed(seed)
    g = torch.randn((n, C) + crop, device=DEV).contiguous(memory_format=mf)
    shapes = [(2, C) + s for s in sps]
    strides = [_cl_strides(s) for s in shapes]
    return crop, sps, shapes, strides, boxes, ind, level, g


@pytest.mark.parametrize("dim", [2, 3])
def test_pyramid_backward_is_the_specified_sum_per_level(dim):
    """mdt_pyramid_roi_align_backward over 4 levels: each level's map equals the restatement of that level's RoIs (clamped roi_level) bit for
    bit, with zero_init 1 and 0, and equals mdt_crop_and_resize_*_backward on that level with the other RoIs' box_ind set to -1"""
    lib = L.load()
    crop, sps, shapes, strides, boxes, ind, level, g = _pyr_setup(dim)
    n, C = boxes.shape[0], shapes[0][1]
    bt, it, lt = (torch.from_numpy(a).to(DEV) for a in (boxes, ind, level))
    gs5 = _strides5(g.stride())
    numel = [int(np.prod(s)) for s in shapes]
    mst = L.i64arr([s for st in strides for s in _strides5(st)])
    dims = _i32([d for s in sps for d in (tuple(s) + (1,) * (3 - len(s)))])
    cz = crop[2] if dim == 3 else 1
    g_flat = g.permute(0, *range(2, dim + 2), 1).contiguous().cpu().numpy().ravel()    # the channels-last storage in memory order

    def call(zero_init):
        def c(o, ws):
            gp = (ctypes.c_void_p * 4)(*o)
            return lib.mdt_pyramid_roi_align_backward(dim, L.ptr(g), L.i64arr(gs5), L.ptr(bt), L.ptr(it), L.ptr(lt), n, 2, crop[0], crop[1], cz, C, gp,
                                                      mst, dims, 4, zero_init, L.i64arr(numel), _sp())
        return c

    outs = _run_guarded(call(1), [4 * m for m in numel], None)
    priors = [torch.randn(m, generator=torch.Generator().manual_seed(m)).float() for m in numel]
    outs0 = _run_prior(call(0), [p.view(torch.uint8).to(DEV) for p in priors])
    for lv in range(4):
        kw = dict(roi_level=level, level=lv, nlevels=4)
        want = _model(g_flat, gs5, boxes, ind, np.zeros(numel[lv], np.float32), _strides5(strides[lv]), shapes[lv], crop, 1, **kw)
        _same_bits(_f32(outs[lv]), want)
        _same_bits(_f32(outs0[lv]), _model(g_flat, gs5, boxes, ind, priors[lv].numpy(), _strides5(strides[lv]), shapes[lv], crop, 0, **kw))
        # the single-map entry point on this level's RoIs gives the same bits
        ind_l = torch.from_numpy(np.where(np.clip(level, 0, 3) == lv, ind, -1).astype(np.int32)).to(DEV)
        one = _run_guarded(_bwd_call(g, gs5, bt, ind_l, crop, _strides5(strides[lv]), shapes[lv], numel[lv], 1), [4 * numel[lv]], None,
                           offsets=(0,))[0]
        assert torch.equal(one, outs[lv])


@pytest.mark.parametrize("dim", [2, 3])
def test_paths_give_the_same_bits(dim):
    """channels-last aligned (vector gather), channels-last 4 bytes off 16 (scalar gather), NCDHW image and crops (scalar gather) and a
    one-level pyramid: the same logical gradient, bit for bit"""
    lib = L.load()
    crop = (7, 7, 3) if dim == 3 else (7, 7)
    shape = (2, 36) + ((16, 16, 12) if dim == 3 else (24, 20))
    mf = CL3 if dim == 3 else torch.channels_last
    boxes, ind = _roi_boxes(30, dim, 2, seed=11)
    bt, it = torch.from_numpy(boxes).to(DEV), torch.from_numpy(ind).to(DEV)
    torch.manual_seed(4)
    g_nc = torch.randn((30, 36) + crop, device=DEV)
    g_cl = g_nc.contiguous(memory_format=mf)
    numel = int(np.prod(shape))
    res = {}
    for name, g, is5, offs in [("cl4", g_cl, _strides5(_cl_strides(shape)), (0,)), ("scalar_mis", g_cl, _strides5(_cl_strides(shape)), (4,)),
                               ("scalar_nc", g_nc, _strides5(torch.empty(shape, device="meta").stride()), (0,))]:
        out = _run_guarded(_bwd_call(g, _strides5(g.stride()), bt, it, crop, is5, shape, numel, 1), [4 * numel], None, offsets=offs)[0]
        res[name] = torch.as_strided(out.view(torch.float32), shape, is5[:dim + 2])
    lt = torch.zeros(30, dtype=torch.int32, device=DEV)
    is5 = _strides5(_cl_strides(shape))
    dims = _i32(tuple(shape[2:]) + (1,) * (5 - len(shape)))
    gp_call = lambda o, ws: lib.mdt_pyramid_roi_align_backward(dim, L.ptr(g_cl), L.i64arr(_strides5(g_cl.stride())), L.ptr(bt), L.ptr(it), L.ptr(lt), 30,
                                                               2, crop[0], crop[1], crop[2] if dim == 3 else 1, 36, (ctypes.c_void_p * 1)(*o),
                                                               L.i64arr(is5), dims, 1, 1, L.i64arr([numel]), _sp())
    res["pyramid"] = torch.as_strided(_run_guarded(gp_call, [4 * numel], None, offsets=(0,))[0].view(torch.float32), shape, is5[:dim + 2])
    for k, v in res.items():
        assert torch.equal(v, res["cl4"]), k


def _stress(dim, boxes, ind, C=8, sp=None, crop=None, g=None, layout="cl"):
    sp = sp or ((12, 10, 8) if dim == 3 else (16, 12))
    crop = crop or ((7, 7, 3) if dim == 3 else (7, 7))
    shape = (2, C) + tuple(sp)
    n = boxes.shape[0]
    cshape = (n, C) + tuple(crop)
    if g is None:
        torch.manual_seed(n)
        g = torch.randn(cshape)
    mf = CL3 if dim == 3 else torch.channels_last
    g = g.to(DEV)
    g = g.contiguous(memory_format=mf) if layout == "cl" else g.contiguous()
    is5 = _strides5(_cl_strides(shape) if layout == "cl" else torch.empty(shape, device="meta").stride())
    gs5 = _strides5(g.stride())
    bt, it = torch.from_numpy(boxes).to(DEV), torch.from_numpy(ind).to(DEV)
    numel = int(np.prod(shape))
    g_mem = (g.permute(0, *range(2, dim + 2), 1) if layout == "cl" else g).contiguous().cpu().numpy().ravel()
    adj = _roi_ref_bwd(g, boxes, ind, crop, shape) if bool(torch.isfinite(g).all()) else None
    got = _check_entry(lambda z: _bwd_call(g, gs5, bt, it, crop, is5, shape, numel, z), g_mem, gs5, boxes, ind, shape, is5, crop, numel * 4, (0, 256),
                       adjoint=adj)
    return torch.as_strided(torch.from_numpy(got), shape, is5[:dim + 2]), shape


@pytest.mark.parametrize("dim", [2, 3])
def test_identical_boxes_pile_up_in_order(dim):
    """512 identical boxes on one batch item: hundreds of terms per voxel, more RoIs than one 256-RoI chunk, all overlapping every tile"""
    box = np.array([0.2, 0.1, 0.7, 0.8] + ([0.3, 0.9] if dim == 3 else []), np.float32)
    boxes = np.tile(box, (512, 1))
    ind = np.zeros(512, np.int32)
    gx, _ = _stress(dim, boxes, ind)
    assert bool((gx[1] == 0).all()) and bool((gx[0] != 0).any())


@pytest.mark.parametrize("dim", [2, 3])
def test_many_overlapping_rois_across_chunks(dim):
    """700 random boxes that all contain the map centre, on both batch items, in both layouts (vector and scalar gather)"""
    rs = np.random.RandomState(dim)
    n = 700
    lo = rs.uniform(0.0, 0.45, size=(n, dim))
    hi = rs.uniform(0.55, 1.0, size=(n, dim))
    cols = [lo[:, 0], lo[:, 1], hi[:, 0], hi[:, 1]] + ([lo[:, 2], hi[:, 2]] if dim == 3 else [])
    boxes = np.stack(cols, 1).astype(np.float32)
    ind = rs.randint(0, 2, size=n).astype(np.int32)
    for layout in ("cl", "nc"):
        _stress(dim, boxes, ind, C=4, layout=layout)


@pytest.mark.parametrize("dim", [2, 3])
def test_border_inverted_crop1_and_bad_box_ind(dim):
    """boxes clamped at the border (lo == hi == size - 1), before the origin, inverted, zero extent, with crop extent 1 on two axes; bad box_ind
    (-1, batch, large) next to good ones, their gradient rows NaN: nothing of them reaches the image"""
    z = lambda a, b: [a, b] if dim == 3 else []
    boxes = np.array([[1.0, 1.0, 1.0, 1.0] + z(1.0, 1.0), [0.9, 0.95, 1.4, 1.3] + z(0.8, 1.6), [-0.6, -0.5, -0.1, -0.2] + z(-0.3, -0.1),
                      [0.8, 0.7, 0.2, 0.1] + z(0.9, 0.3), [0.4, 0.3, 0.4, 0.3] + z(0.5, 0.5), [0.1, 0.2, 0.6, 0.9] + z(0.0, 1.0),
                      [0.7, 0.1, 0.3, 0.6] + z(0.2, 0.8), [0.0, 0.0, 1.0, 1.0] + z(0.0, 1.0), [0.3, 0.3, 0.9, 0.6] + z(0.1, 0.4)], np.float32)
    ind = np.array([0, 1, 0, 1, 0, -1, 2, 1000, 1], np.int32)
    for crop in ([(7, 7, 3), (1, 5, 1), (3, 1, 1)] if dim == 3 else [(7, 7), (1, 5), (4, 1)]):
        torch.manual_seed(1)
        g = torch.randn((9, 8) + crop)
        g[torch.from_numpy((ind < 0) | (ind >= 2))] = float("nan")
        gx, _ = _stress(dim, boxes, ind, crop=crop, g=g)
        assert bool(torch.isfinite(gx).all())


@pytest.mark.parametrize("dim", [2, 3])
def test_inf_gradient_behind_zero_weight_corners(dim):
    """a box whose sample coordinates are all integral (lerp 0: every hi corner has weight 0 and the same voxel as its lo corner): an Inf
    gradient reaches its voxels as +Inf, not as Inf + 0 * Inf = NaN, and no other voxel"""
    # map extent 8, crop 4: scale 2, t = fma(1/16, 8, 2 o) + 1 - 0.5 = 2 o + 1
    box = [0.0625, 0.0625, 1.0625, 1.0625] + ([0.0625, 1.0625] if dim == 3 else [])
    boxes = np.array([box, [0.2, 0.3, 0.6, 0.7] + ([0.1, 0.5] if dim == 3 else [])], np.float32)
    ind = np.array([0, 0], np.int32)
    crop = (4, 4, 4) if dim == 3 else (4, 4)
    tlo, thi, lerp = M.taps(boxes[0, 0], boxes[0, 2], 4, 8)
    assert (lerp == 0).all() and (tlo == thi).all() and tlo.tolist() == [1, 3, 5, 7]
    torch.manual_seed(2)
    g = torch.randn((2, 4) + crop)
    g[0, :, 1, 2] = float("inf")
    gx, _ = _stress(dim, boxes, ind, C=4, sp=(8,) * dim, crop=crop, g=g)
    hit = gx[0, :, 3, 5, 1::2] if dim == 3 else gx[0, :, 3, 5]
    assert bool(torch.isposinf(hit).all()) and not bool(torch.isnan(gx).any())
    assert int(torch.isinf(gx).sum()) == 4 * (4 if dim == 3 else 1)


# ================================================================================================== whole models
def _mrcnn_golden(case):
    sys.path.insert(0, GOLD)
    import detweights
    import golden_inputs as GI
    from test_model_golden import _batch_from_golden
    from medicaldetectiontoolkit_b200 import mrcnn
    cf, model, B = GI.model_case(case)

    def build():
        return GI.tame_(detweights.fill_(mrcnn.net(cf, None)), model).to(DEV)
    g = np.load(os.path.join(GOLD, "model_%s.npz" % case))
    return build, _batch_from_golden(cf, g, B, True, case)


def _mrcnn_2d():
    sys.path.insert(0, GOLD)
    import detweights
    import golden_inputs as GI
    from medicaldetectiontoolkit_b200 import mrcnn
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    cf = make_cf('mrcnn', 2, (128, 128), exp='toy_exp', batch_size=4)

    def build():
        return GI.tame_(detweights.fill_(mrcnn.net(cf, None)), 'mrcnn').to(DEV)
    return build, synthetic_batch(cf, 4, seed=3, with_masks=True)


def _ufrcnn(case):
    sys.path.insert(0, GOLD)
    import make_ufrcnn_golden as G
    from medicaldetectiontoolkit_b200 import ufrcnn as UF
    cf = G.case_cf(case)
    g = np.load(os.path.join(GOLD, "ufrcnn_model_%s.npz" % case))
    return (lambda: G.weights_(UF.net(cf)).to(DEV)), G.batch_from_golden(cf, g, case)


MODELS = {"mrcnn_small": lambda: _mrcnn_golden("mrcnn_small"), "mrcnn_cfg3": lambda: _mrcnn_golden("mrcnn_cfg3"), "mrcnn_2d": _mrcnn_2d,
          "ufrcnn_small": lambda: _ufrcnn("small")}


@pytest.mark.parametrize("case", list(MODELS))
def test_train_steps_are_bit_identical(case, monkeypatch):
    """two train steps from the same weights and batch give bit-identical losses and EVERY parameter gradient, fpn.* included (they receive
    the RoIAlign backward); two runs of three Adam steps give bit-identical parameters"""
    from medicaldetectiontoolkit_b200 import model_utils as mutils
    monkeypatch.setattr(mutils, "SAMPLING", "random")
    build, batch = MODELS[case]()

    def step(net):
        torch.manual_seed(1)
        np.random.seed(1)
        net.zero_grad(set_to_none=True)
        res = net.train_forward(batch)
        res['torch_loss'].backward()
        return float(res['torch_loss'].detach())

    net = build()
    l1 = step(net)
    g1 = {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}
    l2 = step(net)
    g2 = {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}
    assert l1 == l2 and sorted(g1) == sorted(g2)
    assert any(k.startswith("fpn.") for k in g1) and any(float(g1[k].abs().sum()) > 0 for k in g1 if k.startswith("fpn."))
    differ = [k for k in g1 if not torch.equal(g1[k], g2[k])]
    assert not differ, differ
    del net

    def train3():
        net = build()
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        for _ in range(3):
            step(net)
            opt.step()
        return {k: p.detach().clone() for k, p in net.named_parameters()}
    p1, p2 = train3(), train3()
    differ = [k for k in p1 if not torch.equal(p1[k], p2[k])]
    assert not differ, differ
