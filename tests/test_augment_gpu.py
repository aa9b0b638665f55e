"""GPU augmentation ops (csrc/augment.cu through augment.py) against the numpy / scipy oracle: the elastic field, the spatial transform's
data and instance map, the seg-to-box outputs, the validation crop, guarded buffers, determinism, and train steps fed by the augmenter."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import augment as A
from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_precrop_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _guarded as G  # noqa: E402
import augment_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ci(v):
    return (ctypes.c_int * len(v))(*v)


# ------------------------------------------------------------------------------------------------------------------ elastic field
@pytest.mark.parametrize("dim,shape", [(2, (288, 288)), (3, (72, 64, 40))])
@pytest.mark.parametrize("sigma", [30.0, 50.0])
def test_elastic_field_vs_gaussian_filter(dim, shape, sigma):
    from scipy.ndimage import gaussian_filter
    g = torch.Generator(device=DEV).manual_seed(3)
    noise = torch.rand((2, dim) + shape, generator=g, dtype=torch.float64, device=DEV) * 2 - 1
    got = A.elastic_field(noise, [sigma, sigma * 0.9], [1.0, 1.0]).cpu().numpy()
    nz = noise.cpu().numpy()
    for b in range(2):
        for d in range(dim):
            ref = gaussian_filter(nz[b, d], sigma if b == 0 else sigma * 0.9, mode='constant', cval=0)
            # fp64 weights and accumulation, as scipy: the two differ only by summation order and the device's exp (about 3e-15)
            assert np.abs(got[b, d] - ref).max() <= 1e-12 * np.abs(ref).max()
    scaled = A.elastic_field(noise, [sigma, sigma * 0.9], [1500.0, 7.0]).cpu().numpy()
    assert np.array_equal(scaled[0], got[0] * 1500.0) and np.array_equal(scaled[1], got[1] * 7.0)


def test_elastic_field_guarded():
    shape = [40, 36]
    n = 4
    noise = torch.rand([n] + shape, dtype=torch.float64, device=DEV) * 2 - 1
    lib = L.load()
    wsb = lib.mdt_augment_gaussian_workspace_bytes(2, n, _ci(shape))
    sig = (ctypes.c_double * n)(30., 31., 45., 50.)
    sca = (ctypes.c_double * n)(1., 2., 3., 4.)
    out_bytes = n * 40 * 36 * 8
    call = lambda o, ws: lib.mdt_augment_gaussian(2, L.ptr(noise), n, _ci(shape), sig, sca, o[0], ws, wsb, L.stream_ptr())  # noqa: E731
    got = G._run_guarded(call, [out_bytes], wsb)[0].view(torch.float64).view(n, *shape)
    ref = A.elastic_field(noise.view(n, 1, *shape), [30., 31., 45., 50.], [1., 2., 3., 4.]).view(n, *shape)
    assert torch.equal(got, ref)
    sig_bad = (ctypes.c_double * n)(30., 31., 45., 51.)
    assert lib.mdt_augment_gaussian(2, L.ptr(noise), n, _ci(shape), sig_bad, sca, L.ptr(ref), L.ptr(noise), wsb, L.stream_ptr()) == -3


# ------------------------------------------------------------------------------------------------------------------ spatial transform
def _elements(dim, B, src, da, seed, identity=False, scale=None):
    rs = np.random.RandomState(seed)
    prm = A.draw_params(rs, da, dim, B, src)
    if identity:
        prm['flip'][:] = False
        prm['angles'][:] = 0
        prm['scale'][:] = 1
        prm['alpha'][:] = 0
    if scale is not None:
        prm['scale'][:] = scale
    return prm


def _run_spatial(data, seg, prm, dim, patch, da, elastic_on):
    blocks = torch.from_numpy(A.param_blocks(prm, dim, True).view(np.uint8).copy()).to(DEV)
    elastic = None
    if elastic_on:
        g = torch.Generator(device=DEV).manual_seed(prm['noise_seed'])
        noise = torch.rand((data.shape[0], dim, *patch), generator=g, dtype=torch.float64, device=DEV) * 2 - 1
        elastic = A.elastic_field(noise, prm['sigma'], prm['alpha'])
    d, s = A.spatial_transform(torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV), blocks, patch, elastic)
    return d.cpu().numpy(), s.cpu().numpy(), (elastic.cpu().numpy() if elastic is not None else None), blocks


def _coords(prm, b, dim, patch, disp):
    """the op's fp64 coordinates: mesh + displacement, . (R * scale), + centre"""
    c = np.array(np.meshgrid(*[np.arange(p) for p in patch], indexing='ij')).astype(float)
    for d in range(dim):
        c[d] -= (patch[d] - 1) / 2.
        if disp is not None:
            c[d] += disp[b, d]
    m = A.param_blocks(prm, dim, True)['m'][b].reshape(3, 3)[:dim, :dim]
    c = c.reshape(dim, -1).T.dot(m).T.reshape(c.shape)
    for d in range(dim):
        c[d] += prm['centre'][b, d]
    return c


def _near_boundary(c, src):
    """voxels whose coordinate lies within 1e-9 of an order-0 rounding boundary or of the [0, S-1] edge on some axis"""
    near = np.zeros(c.shape[1:], dtype=bool)
    for d in range(c.shape[0]):
        f = c[d] - np.floor(c[d])
        near |= np.abs(f - 0.5) < 1e-9
        near |= (np.abs(c[d]) < 1e-9) | (np.abs(c[d] - (src[d] - 1)) < 1e-9)
    return near


SPATIAL = [
    # name, dim, B, C, src, patch, exp, identity, scale
    ('lidc3d', 3, 2, 1, (156, 156, 96), (128, 128, 64), 'lidc_exp', False, None),
    ('lidc2d', 2, 4, 1, (300, 300), (288, 288), 'lidc_exp', False, None),
    ('toy2d', 2, 4, 1, (320, 320), (320, 320), 'toy_exp', False, None),
    ('odd3d', 3, 2, 3, (41, 37, 29), (33, 35, 27), 'lidc_exp', False, None),
    ('odd2d', 2, 3, 3, (61, 53), (45, 51), 'lidc_exp', False, None),
    ('identity3d', 3, 2, 1, (64, 48, 32), (64, 48, 32), 'lidc_exp', True, None),
    ('identity2d', 2, 2, 2, (64, 48), (64, 48), 'lidc_exp', True, None),
    ('scale1.1_3d', 3, 2, 1, (60, 60, 40), (60, 60, 40), 'lidc_exp', False, 1.1),
    ('scale1.1_2d', 2, 3, 1, (96, 96), (96, 96), 'toy_exp', False, 1.1),
]


@pytest.mark.parametrize("name,dim,B,C,src,patch,exp,identity,scale", SPATIAL, ids=[s[0] for s in SPATIAL])
def test_spatial_transform_vs_oracle(name, dim, B, C, src, patch, exp, identity, scale):
    cf = make_cf('retina_unet', dim, patch, exp=exp)
    cf.n_channels = C
    da = cf.da_kwargs
    batch = synthetic_precrop_batch(cf, src, B, seed=5, empty=())
    data = (batch['data'] * 200 - 50).astype(np.float32)          # an offset, signed range
    prm = _elements(dim, B, src, da, seed=11, identity=identity, scale=scale)
    elastic_on = da['do_elastic_deform'] and not identity
    got, gseg, disp, _ = _run_spatial(data, batch['seg'], prm, dim, list(patch), da, elastic_on)
    tol = 1e-5 * np.abs(data).max()
    n_near_total = 0
    for b in range(B):
        c = _coords(prm, b, dim, patch, disp)
        flip = prm['flip'][b].tolist()
        ref, rseg = O.resample(data[b], batch['seg'][b], flip, c)
        err = np.abs(got[b] - ref).max()
        assert err <= tol, (name, b, err, tol)
        if scale is not None:
            outside = np.zeros(c.shape[1:], dtype=bool)
            for d in range(dim):
                outside |= (c[d] < 0) | (c[d] > src[d] - 1)
            assert outside.mean() > 0.05
        diff = gseg[b, 0] != rseg[0]
        near = _near_boundary(c, src)
        assert not (diff & ~near).any(), (name, b, int((diff & ~near).sum()))
        n_near_total += int((diff & near).sum())
        if identity:
            # every coordinate lies on a half voxel: scipy's rounding rule must be reproduced, not exempted
            assert n_near_total == 0
    print(name, "seg voxels differing at a rounding boundary:", n_near_total)


def test_order0_edge_rule_probe():
    """scipy's order-0 mode='constant' rule, probed: 0 outside [0, S-1], else index floor(q + 0.5) (half rounds up)"""
    from scipy.ndimage import map_coordinates
    a = np.arange(1, 6, dtype=np.float64)
    q = np.array([-0.5, -1e-12, 0.0, 0.5, 1.5, 3.5, 4.0, 4.0 + 1e-12, 4.49])
    got = map_coordinates(a, [q], order=0, mode='constant', cval=0)
    want = [a[int(np.floor(x + 0.5))] if 0 <= x <= 4 else 0 for x in q]
    assert got.tolist() == want


def test_spatial_guarded():
    dim, B, C, src, patch = 3, 2, 2, [21, 19, 13], [17, 15, 11]
    cf = make_cf('retina_unet', dim, patch)
    cf.n_channels = C
    batch = synthetic_precrop_batch(cf, src, B, seed=2, empty=())
    prm = _elements(dim, B, src, cf.da_kwargs, seed=4)
    blocks = torch.from_numpy(A.param_blocks(prm, dim).view(np.uint8).copy()).to(DEV)
    data = torch.from_numpy(batch['data']).to(DEV)
    seg = torch.from_numpy(batch['seg']).to(DEV)
    disp = torch.randn((B, dim, *patch), dtype=torch.float64, device=DEV)
    lib = L.load()
    wsb = lib.mdt_augment_spatial_workspace_bytes(dim, B, C, _ci(src))
    call = lambda o, ws: lib.mdt_augment_spatial(dim, L.ptr(data), L.ptr(seg), B, C, _ci(src), _ci(patch), L.ptr(blocks), L.ptr(disp), o[0],  # noqa
                                                 o[1], ws, wsb, L.stream_ptr())
    vol = int(np.prod(patch))
    got = G._run_guarded(call, [B * C * vol * 4, B * vol], wsb)
    ref_d, ref_s = A.spatial_transform(data, seg, blocks, patch, disp)
    assert torch.equal(got[0].view(torch.float32).view_as(ref_d), ref_d)
    assert torch.equal(got[1].view_as(ref_s), ref_s)
    # no seg
    call = lambda o, ws: lib.mdt_augment_spatial(dim, L.ptr(data), None, B, C, _ci(src), _ci(patch), L.ptr(blocks), None, o[0], None, ws,  # noqa
                                                 wsb, L.stream_ptr())
    G._run_guarded(call, [B * C * vol * 4], wsb)
    assert lib.mdt_augment_spatial(dim, L.ptr(data), L.ptr(seg), B, C, _ci(src), _ci(patch), L.ptr(blocks), None, L.ptr(ref_d), None,
                                   L.ptr(disp), wsb, L.stream_ptr()) == -1


# ------------------------------------------------------------------------------------------------------------------ seg to boxes
@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("class_specific", [False, True])
def test_seg_to_boxes_guarded_vs_oracle(dim, class_specific):
    patch = [40, 36, 24][:dim]
    cf = make_cf('mrcnn', dim, patch)
    batch = synthetic_precrop_batch(cf, patch, 4, seed=9, empty=(2,))
    seg = torch.from_numpy(batch['seg']).to(DEV)
    ct = batch['class_target']
    lut = torch.from_numpy(A.label_lut(ct, class_specific)).to(DEV)
    nm = max(len(c) for c in ct)
    lib = L.load()
    vol = int(np.prod(patch))
    call = lambda o, ws: lib.mdt_augment_seg_to_boxes(dim, L.ptr(seg), 4, _ci(patch), L.ptr(lut), nm, o[0], o[1], o[2], L.stream_ptr())  # noqa
    st, sseg, masks = G._run_guarded(call, [4 * 255 * 7 * 4, 4 * vol, 4 * nm * vol], None)
    st = st.view(torch.int32).view(4, 255, 7).cpu().numpy()
    masks = masks.view(4, nm, *patch).cpu().numpy()
    bb, labels, rm = A.boxes_from_stats(st, ct, dim, masks)
    want = O.seg_to_boxes(batch['seg'], ct, dim, class_specific)
    assert np.array_equal(sseg.view(4, 1, *patch).cpu().numpy(), want['seg'])
    for b in range(4):
        assert np.array_equal(np.asarray(bb[b]), np.asarray(want['bb_target'][b]))
        assert np.array_equal(labels[b], want['roi_labels'][b])
        assert np.array_equal(rm[b], want['roi_masks'][b])
    assert bb[2] == [] and labels[2].tolist() == [-1]


# ------------------------------------------------------------------------------------------------------------------ augmenter
def _oracle_batch(cf, batch, seed, with_masks):
    """the whole chain on the host: oracle draws, the device noise of the same seed through scipy's gaussian_filter, mirror +
    map_coordinates, seg to boxes"""
    dim = cf.dim
    P = cf.patch_size[:dim]
    B = batch['data'].shape[0]
    src = batch['data'].shape[2:]
    elems, nseed = O.draw_params(np.random.RandomState([seed, 0]), cf.da_kwargs, dim, B, src)
    noise = None
    if nseed is not None:
        g = torch.Generator(device=DEV).manual_seed(nseed)
        noise = (torch.rand((B, dim, *P), generator=g, dtype=torch.float64, device=DEV) * 2 - 1).cpu().numpy()
    data, seg, coords = [], [], []
    for b, e in enumerate(elems):
        c = O.coordinates(e, P, None if noise is None else noise[b])
        d, s = O.resample(batch['data'][b], batch['seg'][b], e['flip'], c)
        data.append(d)
        seg.append(s)
        coords.append(c)
    res = O.seg_to_boxes(np.stack(seg), batch['class_target'], dim, cf.class_specific_seg_flag, with_masks)
    res['data'] = np.stack(data)
    res['coords'] = coords
    return res


@pytest.mark.parametrize("dim", [3, 2])
def test_augmenter_end_to_end(dim):
    patch, src = ((128, 128, 64), (156, 156, 96)) if dim == 3 else ((288, 288), (300, 300))
    cf = make_cf('mrcnn', dim, patch)
    cf.class_specific_seg_flag = True
    batch = synthetic_precrop_batch(cf, src, 3, seed=1, empty=(1,))
    out = A.Augmenter(cf, seed=6, rank=0, with_masks=True)(batch)
    want = _oracle_batch(cf, batch, 6, True)
    assert out['data'].dtype == torch.float32 and out['data'].is_cuda and out['seg'].dtype == torch.uint8
    # data: the 2D elastic field agrees with scipy's to about 1e-15 of its size, so it moves the coordinates by far less than the fp32
    # spline's own error and both dims meet the same bound
    tol = 1e-5 * np.abs(batch['data']).max()
    assert np.abs(out['data'].cpu().numpy() - want['data']).max() <= tol
    gseg = out['seg'].cpu().numpy()
    # the seg, and with it every box, label and mask, equal the oracle's except at rounding boundaries
    near = np.stack([_near_boundary(c, src) for c in want['coords']])[:, None]
    assert not ((gseg != want['seg']) & ~near).any()
    if not ((gseg != want['seg']) & near).any():
        for b in range(3):
            assert np.array_equal(np.asarray(out['bb_target'][b]), np.asarray(want['bb_target'][b]))
            assert np.array_equal(out['roi_labels'][b], want['roi_labels'][b])
            assert np.array_equal(out['roi_masks'][b], want['roi_masks'][b])
    # always: boxes / labels / masks / relabelled seg equal the oracle applied to the op's own warped instance map
    raw = _raw_warp(cf, batch, 6)
    ref = O.seg_to_boxes(raw, batch['class_target'], dim, True)
    assert np.array_equal(gseg, ref['seg'])
    for b in range(3):
        assert np.array_equal(np.asarray(out['bb_target'][b]), np.asarray(ref['bb_target'][b]))
        assert np.array_equal(out['roi_labels'][b], ref['roi_labels'][b])
        assert np.array_equal(out['roi_masks'][b], ref['roi_masks'][b])
    assert out['bb_target'][1] == [] and out['roi_labels'][1].tolist() == [-1] and out['roi_masks'][1].shape == (1, 1) + tuple(patch)


def _raw_warp(cf, batch, seed):
    """the op's warped instance map (before relabelling) for the Augmenter's first batch of this seed"""
    dim = cf.dim
    P = cf.patch_size[:dim]
    B = batch['data'].shape[0]
    prm = A.draw_params(np.random.RandomState([seed, 0]), cf.da_kwargs, dim, B, batch['data'].shape[2:])
    _, s, _, _ = _run_spatial(batch['data'], batch['seg'], prm, dim, list(P), cf.da_kwargs, cf.da_kwargs['do_elastic_deform'])
    return s


def test_validation_crop_equals_slicing():
    cf = make_cf('retina_unet', 3, (64, 48, 32))
    batch = synthetic_precrop_batch(cf, (77, 60, 41), 3, seed=3, empty=(0,))
    out = A.Augmenter(cf, is_training=False, seed=0, rank=0)(batch)
    assert np.array_equal(out['data'].cpu().numpy(), O.center_crop(batch['data'], (64, 48, 32)))
    want = O.seg_to_boxes(np.ascontiguousarray(O.center_crop(batch['seg'], (64, 48, 32))), batch['class_target'], 3, False, False)
    assert np.array_equal(out['seg'].cpu().numpy(), want['seg'])
    for b in range(3):
        assert np.array_equal(np.asarray(out['bb_target'][b]), np.asarray(want['bb_target'][b]))
        assert np.array_equal(out['roi_labels'][b], want['roi_labels'][b])


@pytest.mark.parametrize("dim", [2, 3])
def test_augmenter_deterministic(dim):
    patch, src = ((64, 64, 32), (80, 76, 40)) if dim == 3 else ((96, 96), (110, 104))
    cf = make_cf('mrcnn', dim, patch)
    cf.da_kwargs['do_elastic_deform'] = True
    batch = synthetic_precrop_batch(cf, src, 4, seed=2, empty=(3,))
    runs = []
    for _ in range(2):
        aug = A.Augmenter(cf, seed=13, rank=0, with_masks=True)
        runs.append([aug(batch), aug(batch)])
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a['data'], b['data']) and torch.equal(a['seg'], b['seg'])
        for k in ('bb_target', 'roi_labels', 'roi_masks'):
            for x, y in zip(a[k], b[k]):
                assert np.array_equal(np.asarray(x), np.asarray(y))
    assert not torch.equal(runs[0][0]['data'], runs[0][1]['data'])
    other = A.Augmenter(cf, seed=13, rank=1)(batch)
    assert not torch.equal(other['data'], runs[0][0]['data'])


@pytest.mark.parametrize("model", ["retina_unet", "mrcnn"])
def test_train_step_fed_by_augmenter(model):
    """a train step at 128 x 128 x 64 fed by the augmenter (one element without foreground) gives the loss of the same batch as host numpy"""
    import importlib
    mod = importlib.import_module("medicaldetectiontoolkit_b200." + model)
    cf = make_cf(model, 3, (128, 128, 64))
    batch = synthetic_precrop_batch(cf, (156, 156, 96), 2, seed=4, empty=(1,))
    aug = A.Augmenter(cf, seed=0, rank=0, with_masks=(model == 'mrcnn'))(batch)
    host = dict(aug, data=aug['data'].cpu().numpy(), seg=aug['seg'].cpu().numpy())
    torch.manual_seed(0)
    net = mod.net(cf, None).to(DEV)
    net.train()
    losses = []
    for b in (aug, host):
        torch.manual_seed(1)
        np.random.seed(1)
        res = net.train_forward(b)
        losses.append(res['torch_loss'].detach().cpu())
        assert np.isfinite(res['monitor_values']['loss'])
    assert torch.equal(losses[0], losses[1])
