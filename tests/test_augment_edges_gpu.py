"""The augmentation kernels (csrc/augment.cu) and the component masks of csrc/seg_rois.cu at their edges, against plain references:
  - the elastic field against scipy.ndimage.gaussian_filter to 1e-12 of max|ref| per field: the patches that run elastic deformation, the
    radius limits, windows clipped on both sides, the 3D ping-pong, the field-count limit and guarded buffers;
  - the spatial transform against mirror + map_coordinates on the op's own fp64 coordinates: every flip combination, patches larger than
    the source (coordinates past the pad clamp), sources 1-3 voxels thin, 2 and 5 channels, non-integer crop centres, 3D rotation about
    all axes, a general matrix, an elastic 3D warp and the no-seg path;
  - seg to boxes bit for bit against the restated statistics and the oracle, on warps that straddle elements, all 255 ids, 32 groups per
    warp, one group per warp and 64 elements;
  - the component masks of more than 65535 components (past the grid-y limit of the mask launch), vectorised and scalar.
The fixtures and the restated statistics come from test_augment_edges_cpu.py, which checks on the host that they can fail."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

from medicaldetectiontoolkit_b200 import _lib as L
from medicaldetectiontoolkit_b200 import augment as A
from medicaldetectiontoolkit_b200.configs import make_cf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _guarded as G  # noqa: E402
import _seg_rois_oracle as R  # noqa: E402
import augment_oracle as O  # noqa: E402
import test_augment_edges_cpu as EC  # noqa: E402
import test_augment_gpu as TAG  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = 12                     # the spline's edge padding: coordinates are clamped to [-PAD, S - 1 + PAD]


def _ci(v):
    return (ctypes.c_int * len(v))(*[int(x) for x in v])


def _cd(v):
    return (ctypes.c_double * len(v))(*[float(x) for x in v])


# ------------------------------------------------------------------------------------------------------------------ elastic field
def _radius(sigma):
    return int(4.0 * sigma + 0.5)


def _noise(n, shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand((n,) + tuple(shape), generator=g, dtype=torch.float64, device=DEV) * 2 - 1


def _gauss_call(noise, sigma, alpha):
    """-> (call(out_ptrs, ws_ptr) of mdt_augment_gaussian with one sigma and alpha per field of noise [n, *shape], workspace bytes)"""
    lib = L.load()
    n, shape = len(sigma), list(noise.shape[1:])
    wsb = lib.mdt_augment_gaussian_workspace_bytes(len(shape), n, _ci(shape))
    sig, sca = _cd(sigma), _cd(alpha)
    return (lambda o, ws: lib.mdt_augment_gaussian(len(shape), L.ptr(noise), n, _ci(shape), sig, sca, o[0], ws, wsb, L.stream_ptr())), wsb


def _gauss(noise, sigma, alpha, guarded=False):
    call, wsb = _gauss_call(noise, sigma, alpha)
    if guarded:
        out = G._run_guarded(call, [noise.numel() * 8], wsb)[0].view(torch.float64)
    else:
        out = torch.empty_like(noise)
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
        L.check(call([L.ptr(out)], L.ptr(ws)))
    return out.view(noise.shape).cpu().numpy()


def _check_fields(name, got, noise, sigma, alpha):
    """every field within 1e-12 of max|ref| of alpha * gaussian_filter(noise, sigma, mode='constant', cval=0); prints the worst ratio"""
    nz = noise.cpu().numpy()
    worst = 0.0
    for f in range(len(sigma)):
        ref = gaussian_filter(nz[f], sigma[f], mode='constant', cval=0) * alpha[f]
        ratio = float(np.abs(got[f] - ref).max() / np.abs(ref).max())
        assert ratio <= EC.ELASTIC_BOUND, (name, f, sigma[f], ratio)
        worst = max(worst, ratio)
    print("elastic %s: worst max|err| / max|ref| %.2e" % (name, worst))
    return worst


ELASTIC_PATCHES = [
    # name, shape, n fields (pet_ct 2D: batch 20 x 2 axes; toy 2D: batch 8 x 2 axes; lidc-sized 3D: 1 x 3 axes at sigma 50)
    ('petct2d', (288, 288), 40),
    ('toy2d', (320, 320), 16),
    ('3d_128x128x64', (128, 128, 64), 3),
]


@pytest.mark.parametrize("name,shape,n", ELASTIC_PATCHES, ids=[e[0] for e in ELASTIC_PATCHES])
def test_elastic_field_at_patch_shapes(name, shape, n):
    rs = np.random.RandomState(n)
    if len(shape) == 3:
        sigma, alpha = [50.0] * n, [1500.0, 700.0, 1.0]           # noise -> out -> tmp -> out
    else:
        sigma, alpha = rs.uniform(30, 50, n), rs.uniform(0, 1500, n)
        sigma[:2] = 30.0, 50.0
    noise = _noise(n, shape, 7)
    _check_fields(name, _gauss(noise, sigma, alpha), noise, sigma, alpha)


def test_elastic_field_radius_limits():
    """radius 200 (the largest) from sigma 49.875 and 50.12, radius 0 (the field is the noise times alpha) and radius 1; sigma 50.125
    (radius 201) is refused and leaves the output bytes as they were"""
    shape = (37, 41)
    sigma, alpha = [49.875, 50.12, 0.1, 0.2], [3.0, 1500.0, 2.5, 900.0]
    assert [_radius(s) for s in sigma] == [200, 200, 0, 1]
    noise = _noise(len(sigma), shape, 1)
    got = _gauss(noise, sigma, alpha)
    _check_fields('radius_limits', got, noise, sigma, alpha)
    assert np.array_equal(got[2], noise[2].cpu().numpy() * alpha[2])
    bad = [30.0, 50.125, 40.0]
    assert _radius(50.125) == 201
    call, wsb = _gauss_call(noise[:3], bad, alpha[:3])
    for run in G._run_guarded_all(call, [3 * 37 * 41 * 8], wsb, expect=-3):
        assert bool((run[0] == G.POISON).all())


@pytest.mark.parametrize("shape", [(9, 1), (1, 7), (5, 1, 3), (12, 10, 2)])
def test_elastic_field_windows_clipped_on_both_sides(shape):
    """every radius larger than every extent, an extent-1 axis among them (that axis multiplies by the centre weight only)"""
    sigma, alpha = [3.3, 10.0, 50.0], [1.0, 300.0, 1500.0]
    assert min(_radius(s) for s in sigma) > max(shape)
    noise = _noise(3, shape, 2)
    _check_fields('clipped_%s' % 'x'.join(map(str, shape)), _gauss(noise, sigma, alpha), noise, sigma, alpha)


def test_elastic_field_count_limit():
    """1024 fields, each with its own sigma (radius 0 to 200) and alpha, are accepted; 1025 are refused and leave the output untouched"""
    shape = (6, 5)
    rs = np.random.RandomState(4)
    sigma, alpha = np.linspace(0.1, 50.0, 1024), rs.uniform(0, 1500, 1024)
    noise = _noise(1025, shape, 3)
    _check_fields('n1024', _gauss(noise[:1024], sigma, alpha), noise[:1024], sigma, alpha)
    call, wsb = _gauss_call(noise, np.append(sigma, 30.0), np.append(alpha, 1.0))
    assert wsb > 0
    for run in G._run_guarded_all(call, [1025 * 30 * 8], wsb, expect=-1):
        assert bool((run[0] == G.POISON).all())


@pytest.mark.parametrize("shape,n", [((40, 36), 40), ((24, 20, 16), 6)])
def test_elastic_field_guarded(shape, n):
    """exact-size poisoned output and workspace: 2D ends in out from tmp, 3D goes noise -> out -> tmp -> out"""
    rs = np.random.RandomState(n)
    sigma, alpha = rs.uniform(30, 50, n), rs.uniform(0, 1500, n)
    noise = _noise(n, shape, 5)
    _check_fields('guarded_%dd' % len(shape), _gauss(noise, sigma, alpha, guarded=True), noise, sigma, alpha)


# ------------------------------------------------------------------------------------------------------------------ spatial transform
def _source(B, C, S, seed):
    """signed, offset fp32 data and per-voxel random instance ids (so that every order-0 index is checked)"""
    rs = np.random.RandomState(seed)
    data = (rs.rand(B, C, *S) * 200 - 50).astype(np.float32)
    seg = rs.randint(0, 10, size=(B, 1) + tuple(S)).astype(np.uint8)
    return data, seg


def _blocks(ms, centres, flips):
    """mdt_augment_params per element from dim x dim matrices (row-vector convention: q_j = sum_d c_d m[d, j]), centres and flips"""
    blocks = np.zeros(len(ms), dtype=A.PARAMS_DTYPE)
    for b, (m, c, f) in enumerate(zip(ms, centres, flips)):
        dim = len(c)
        full = np.identity(3)
        full[:dim, :dim] = m
        blocks['m'][b] = full.reshape(9)
        blocks['centre'][b, :dim] = c
        blocks['flip'][b, :dim] = [int(x) for x in f]
    return blocks


def _coords(blocks, b, patch, disp):
    """the op's fp64 coordinates: mesh + displacement, . m, + centre"""
    dim = len(patch)
    c = np.array(np.meshgrid(*[np.arange(p) for p in patch], indexing='ij')).astype(float)
    for d in range(dim):
        c[d] -= (patch[d] - 1) / 2.
        if disp is not None:
            c[d] += disp[b, d]
    c = c.reshape(dim, -1).T.dot(blocks['m'][b].reshape(3, 3)[:dim, :dim]).T.reshape(c.shape)
    for d in range(dim):
        c[d] += blocks['centre'][b, d]
    return c


def _check_spatial(name, data, seg, blocks, patch, elastic=None, coords=None, exact=()):
    """mdt_augment_spatial against O.resample on every element: data within 1e-5 of max|data|, the instance map equal except within 1e-9
    of a rounding boundary (exactly equal for the elements in `exact`).  elastic: device displacement [B, dim, *P]; coords: the reference
    coordinates per element (default: the op's own).  -> (data, seg, coordinates per element)"""
    dim = len(patch)
    src = data.shape[2:]
    dev_blocks = torch.from_numpy(blocks.view(np.uint8).copy()).to(DEV)
    got, gseg = A.spatial_transform(torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV), dev_blocks, list(patch), elastic)
    got, gseg = got.cpu().numpy(), gseg.cpu().numpy()
    disp = elastic.cpu().numpy() if elastic is not None else None
    tol = 1e-5 * np.abs(data).max()
    cs, n_near = [], 0
    for b in range(data.shape[0]):
        c = coords[b] if coords is not None else _coords(blocks, b, patch, disp)
        ref, rseg = O.resample(data[b], seg[b], blocks['flip'][b, :dim].tolist(), c)
        err = np.abs(got[b] - ref).max()
        assert err <= tol, (name, b, err, tol)
        diff = gseg[b, 0] != rseg[0]
        if b in exact:
            assert not diff.any(), (name, b, int(diff.sum()))
        near = TAG._near_boundary(c, src)
        assert not (diff & ~near).any(), (name, b, int((diff & ~near).sum()))
        n_near += int(diff.sum())
        cs.append(c)
    print("spatial %s: seg voxels differing at a rounding boundary: %d" % (name, n_near))
    return got, gseg, cs


def _rot(dim, angles, scale):
    return A.rotation_matrix(dim, angles) * scale


GEOM = {2: ((37, 29), (31, 27)), 3: ((23, 19, 13), (21, 17, 11))}


@pytest.mark.parametrize("dim", [2, 3])
def test_spatial_every_flip_combination(dim):
    S, P = GEOM[dim]
    flips = list(np.ndindex(*([2] * dim)))
    B = len(flips)
    data, seg = _source(B, 1, S, dim)
    m = _rot(dim, (0.3, 0.2, -0.5), 0.93)
    blocks = _blocks([m] * B, [[s / 2. + o for s, o in zip(S, (0.37, -0.21, 0.15))]] * B, flips)
    assert sorted(map(tuple, blocks['flip'][:, :dim].tolist())) == sorted(flips)
    _check_spatial('flips%dd' % dim, data, seg, blocks, P)


@pytest.mark.parametrize("dim", [2, 3])
def test_spatial_patch_larger_than_source(dim):
    """scale 0.8 and a rotation over a patch four to five times the source: coordinates reach past the pad on both sides of every axis"""
    S, P = ((20, 17), (80, 72)) if dim == 2 else ((12, 10, 8), (64, 60, 56))
    data, seg = _source(2, 1, S, 10 + dim)
    m = _rot(dim, (0.4, 0.5, 0.7) if dim == 3 else (0.4, 0, 0), 0.8)
    blocks = _blocks([m, m], [[s / 2. for s in S]] * 2, [[False] * dim, [True] * dim])
    _, _, cs = _check_spatial('larger%dd' % dim, data, seg, blocks, P)
    for c in cs:
        for d in range(dim):
            assert (c[d] > S[d] - 1 + PAD).mean() > 0.05 and (c[d] < -PAD).mean() > 0.05, (d, (c[d] > S[d] - 1 + PAD).mean(), (c[d] < -PAD).mean())


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("thin", [1, 2, 3])
def test_spatial_thin_source(dim, thin):
    """a source 1, 2 or 3 voxels thin on one axis: the 4-tap window spans the whole padded line, and the order-0 rule's [0, S - 1] is one to
    three voxels.  Element 0 is rotated; element 1 (flipped) samples integer coordinates that include 0 .. S - 1 on the thin axis, so its
    instance map must equal the rule's exactly"""
    if dim == 2:
        S, P, ax = (thin, 23), (9, 19), 0
    else:
        S, P, ax = (17, 15, thin), (15, 13, 5), 2
    data, seg = _source(2, 1, S, 20 + thin)
    ident = np.identity(dim)
    centre1 = [0.0 if d == ax else float(S[d] // 2) for d in range(dim)]
    blocks = _blocks([_rot(dim, (0.35, 0.1, 0.6), 1.02), ident], [[s / 2. + 0.3 for s in S], centre1], [[False] * dim, [True] * dim])
    _, gseg, cs = _check_spatial('thin%dd_%d' % (dim, thin), data, seg, blocks, P, exact=(1,))
    assert set(np.unique(cs[1][ax])) >= set(range(thin)) and gseg[1].any()


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("C", [2, 5])
def test_spatial_channels(dim, C):
    S, P = ((45, 39), (41, 33)) if dim == 2 else ((25, 21, 15), (19, 17, 13))
    data, seg = _source(3, C, S, 30 + C)
    rs = np.random.RandomState(C)
    ms = [_rot(dim, rs.uniform(0, 2 * np.pi, 3), rs.uniform(0.8, 1.1)) for _ in range(3)]
    centres = [[s / 2. + rs.uniform(-2, 2) for s in S] for _ in range(3)]
    blocks = _blocks(ms, centres, rs.rand(3, dim) < 0.5)
    got, _, _ = _check_spatial('channels%dd_C%d' % (dim, C), data, seg, blocks, P)
    assert all(not np.array_equal(got[:, 0], got[:, k]) for k in range(1, C))


@pytest.mark.parametrize("dim", [2, 3])
def test_spatial_random_crop_centres(dim):
    """the random_crop=True draws (non-integer centres), with the config's own elastic field in 2D"""
    S, P = ((110, 104), (96, 96)) if dim == 2 else ((80, 76, 40), (64, 64, 32))
    cf = make_cf('retina_unet', dim, P)
    da = dict(cf.da_kwargs, random_crop=True, rand_crop_dist=tuple(p / 2. - 3 for p in P))
    prm = A.draw_params(np.random.RandomState(40 + dim), da, dim, 3, S)
    assert (prm['centre'] != np.floor(prm['centre'])).all()
    elastic = None
    if da['do_elastic_deform']:
        noise = torch.rand((3, dim, *P), generator=torch.Generator(device=DEV).manual_seed(prm['noise_seed']), dtype=torch.float64,
                           device=DEV) * 2 - 1
        elastic = A.elastic_field(noise, prm['sigma'], prm['alpha'])
    data, seg = _source(3, 1, S, 40 + dim)
    _check_spatial('random_crop%dd' % dim, data, seg, A.param_blocks(prm, dim, True), P, elastic)


def test_spatial_3d_rotation_about_every_axis():
    S, P = (40, 36, 28), (32, 30, 24)
    m = _rot(3, (0.7, -0.5, 1.2), 1.05)
    assert (np.abs(m) > 0.1).all()                                    # every output axis mixes every input axis
    data, seg = _source(2, 1, S, 50)
    blocks = _blocks([m, m], [[20.4, 17.7, 14.2]] * 2, [[False, False, False], [True, False, True]])
    _check_spatial('rot_xyz', data, seg, blocks, P)


@pytest.mark.parametrize("dim", [2, 3])
def test_spatial_general_matrix(dim):
    """shear and anisotropic scale, not through rotation_matrix: q_j = sum_d c_d m[d, j] with m far from symmetric"""
    S, P = GEOM[dim]
    rs = np.random.RandomState(60 + dim)
    ms = [np.identity(dim) + 0.4 * rs.randn(dim, dim) + np.triu(np.full((dim, dim), 0.5), 1) for _ in range(2)]
    off = ~np.eye(dim, dtype=bool)
    for m in ms:
        assert np.abs(m - m.T)[off].min() > 0.15                      # the transposed convention would move every voxel
    data, seg = _source(2, 1, S, 60 + dim)
    blocks = _blocks(ms, [[s / 2. + 0.41 for s in S]] * 2, [[False] * dim, [True] + [False] * (dim - 1)])
    _check_spatial('general%dd' % dim, data, seg, blocks, P)


def test_spatial_3d_elastic_vs_oracle_coordinates():
    """a 3D elastic warp: the reference coordinates come from O.coordinates (scipy's gaussian_filter of the same device noise), not from
    the op's field"""
    S, P = (48, 44, 32), (40, 36, 28)
    B = 2
    rs = np.random.RandomState(70)
    elems = [{'sigma': s, 'alpha': a, 'centre': [x / 2. + rs.uniform(-3, 3) for x in S], 'flip': f}
             for s, a, f in zip((8.0, 11.5), (1000.0, 1500.0), ([False, True, False], [True, True, True]))]
    ms = [_rot(3, rs.uniform(0, 2 * np.pi, 3), rs.uniform(0.8, 1.1)) for _ in range(B)]
    noise = _noise(B * 3, P, 71).view(B, 3, *P)
    elastic = A.elastic_field(noise, [e['sigma'] for e in elems], [e['alpha'] for e in elems])
    nz = noise.cpu().numpy()
    coords = [O.coordinates(e, P, nz[b], matrix=ms[b]) for b, e in enumerate(elems)]
    assert np.abs(elastic.cpu().numpy()).max() > 1.0
    data, seg = _source(B, 1, S, 70)
    blocks = _blocks(ms, [e['centre'] for e in elems], [e['flip'] for e in elems])
    _check_spatial('elastic3d', data, seg, blocks, P, elastic, coords=coords)


def test_spatial_no_seg_guarded_2d():
    """seg = seg_out = NULL through exact-size poisoned buffers: the data equal the seg path's bit for bit"""
    dim, B, C, S, P = 2, 3, 2, (45, 39), (41, 33)
    rs = np.random.RandomState(80)
    data, seg = _source(B, C, S, 80)
    blocks = _blocks([_rot(2, (rs.uniform(0, 6),), rs.uniform(0.8, 1.1)) for _ in range(B)], [[s / 2. + 0.3 for s in S]] * B,
                     rs.rand(B, dim) < 0.5)
    elastic = A.elastic_field(_noise(B * dim, P, 81).view(B, dim, *P), [30.0, 41.0, 50.0], [1500.0, 800.0, 20.0])
    got, _, _ = _check_spatial('noseg2d', data, seg, blocks, P, elastic)
    lib = L.load()
    data_d = torch.from_numpy(data).to(DEV)
    dev_blocks = torch.from_numpy(blocks.view(np.uint8).copy()).to(DEV)
    wsb = lib.mdt_augment_spatial_workspace_bytes(dim, B, C, _ci(S))
    call = lambda o, ws: lib.mdt_augment_spatial(dim, L.ptr(data_d), None, B, C, _ci(S), _ci(P), L.ptr(dev_blocks), L.ptr(elastic), o[0],  # noqa
                                                 None, ws, wsb, L.stream_ptr())
    out = G._run_guarded(call, [B * C * int(np.prod(P)) * 4], wsb)[0]
    assert np.array_equal(out.view(torch.float32).view(B, C, *P).cpu().numpy(), got)


# ------------------------------------------------------------------------------------------------------------------ seg to boxes
@pytest.mark.parametrize("with_masks", [True, False])
@pytest.mark.parametrize("name", sorted(EC.box_cases()))
def test_seg_to_boxes_edges(name, with_masks):
    """raw statistics bit for bit against the restated rule; relabelled seg, boxes, labels and masks against O.seg_to_boxes; class-specific
    relabelling with masks, binary without (masks NULL, n_mask_ids 0)"""
    dim, seg, ct = EC.box_cases()[name]
    B, P = seg.shape[0], list(seg.shape[2:])
    vol = int(np.prod(P))
    if name in EC.STRADDLING:
        assert vol % 32 != 0 and EC.straddling_runs(seg) > 0
    nm = max(len(c) for c in ct) if with_masks else 0
    seg_d = torch.from_numpy(seg).to(DEV)
    lut = torch.from_numpy(A.label_lut(ct, with_masks)).to(DEV)
    lib = L.load()
    call = lambda o, ws: lib.mdt_augment_seg_to_boxes(dim, L.ptr(seg_d), B, _ci(P), L.ptr(lut), nm, o[0], o[1], o[2], L.stream_ptr())  # noqa
    st, sseg, masks = G._run_guarded(call, [B * 255 * 7 * 4, B * vol, B * nm * vol if with_masks else None], None)
    st = st.view(torch.int32).view(B, 255, 7).cpu().numpy()
    assert np.array_equal(st, EC.stats_of(seg))
    want = O.seg_to_boxes(seg, ct, dim, with_masks, with_masks)
    assert np.array_equal(sseg.view(B, 1, *P).cpu().numpy(), want['seg'])
    if with_masks:
        masks = masks.view(B, nm, *P).cpu().numpy()
        assert np.array_equal(masks, np.stack([seg[:, 0] == k for k in range(1, nm + 1)], 1).astype(np.uint8))
    bb, labels, rm = A.boxes_from_stats(st, ct, dim, masks)
    for b in range(B):
        assert np.array_equal(np.asarray(bb[b]), np.asarray(want['bb_target'][b]))
        assert np.array_equal(labels[b], want['roi_labels'][b])
        if with_masks:
            assert np.array_equal(rm[b], want['roi_masks'][b])


def test_seg_to_boxes_refusals():
    """n_mask_ids = 256 (with and without masks) and masks with n_mask_ids = 0 are refused and leave every output as it was"""
    dim, seg, ct = EC.box_cases()['7x9']
    B, P = seg.shape[0], [7, 9]
    seg_d = torch.from_numpy(seg).to(DEV)
    lut = torch.from_numpy(A.label_lut(ct, True)).to(DEV)
    lib = L.load()
    for nm, mask_bytes in ((256, B * 256 * 63), (256, None), (0, B * 63)):
        call = lambda o, ws: lib.mdt_augment_seg_to_boxes(dim, L.ptr(seg_d), B, _ci(P), L.ptr(lut), nm, o[0], o[1], o[2],  # noqa: E731
                                                          L.stream_ptr())
        for run in G._run_guarded_all(call, [B * 255 * 7 * 4, B * 63, mask_bytes], None, expect=-1):
            assert all(o is None or bool((o == G.POISON).all()) for o in run), (nm, mask_bytes)


# ------------------------------------------------------------------------------------------------------------------ ROI masks past grid y
def _checkerboard(B, P):
    """face-isolated foreground: every voxel of even coordinate sum, one component each"""
    return np.broadcast_to(np.indices(P).sum(0) % 2 == 0, (B, 1) + P).astype(np.uint8).copy()


@pytest.mark.parametrize("P,B,label_offset", [((16, 16, 4), 140, 0), ((15, 15, 5), 120, 0), ((16, 16, 4), 140, 4)],
                         ids=["vec", "odd_volume", "label_ptr_16n+4"])
def test_seg_rois_masks_past_grid_y(P, B, label_offset):
    """more than 65535 components over 120-140 elements: components, elem_first, boxes and masks equal scipy.ndimage.label's; the
    vectorised mask kernel (volume a multiple of 4, 16-byte aligned labels) and the scalar one (odd volume, or labels 4 bytes past 16)"""
    V = int(np.prod(P))
    seg = _checkerboard(B, P)
    ct = [0] * B
    label, first, stats, _ = A.seg_rois(torch.from_numpy(seg).to(DEV), torch.zeros(B, dtype=torch.int32, device=DEV), False)
    first_h = first.cpu().numpy()
    K = int(first_h[-1])
    assert K > 65535
    lab = label
    if label_offset:
        buf = torch.empty(B * V + label_offset // 4, dtype=torch.int32, device=DEV)
        buf[label_offset // 4:] = label.view(-1)
        lab = buf[label_offset // 4:]
    assert lab.data_ptr() % 16 == label_offset
    vectorised = V % 4 == 0 and lab.data_ptr() % 16 == 0
    assert vectorised == (label_offset == 0 and P == (16, 16, 4))
    lib = L.load()
    call = lambda o, ws: lib.mdt_seg_rois_masks(3, L.ptr(lab), B, _ci(P), L.ptr(first), K, o[0], L.stream_ptr())  # noqa: E731
    masks = G._run_guarded(call, [K * V], None, offsets=(0,))[0].view(K, *P).cpu().numpy()
    want = R.seg_rois(seg, ct, 3, False)
    label_h = label.cpu().numpy()
    for b in range(B):
        clusters, n = want['components'][b]
        assert first_h[b + 1] - first_h[b] == n
        assert np.array_equal(label_h[b], np.where(clusters > 0, clusters - 1 + first_h[b], -1))
    bb, labels, rm = A.boxes_from_rois(first_h, stats.cpu().numpy(), ct, 3, masks)
    for b in range(B):
        assert np.array_equal(np.asarray(bb[b]), np.asarray(want['bb_target'][b]))
        assert np.array_equal(labels[b], want['roi_labels'][b])
        assert np.array_equal(rm[b], want['roi_masks'][b])
