"""Host-side self-checks of the augmentation edge suite (test_augment_edges_gpu.py): the bound on the elastic field is met by the kernel's own
summation order in fp64 and missed by a field with fp32 weights, and the seg-to-box fixtures put voxels of two elements that carry the same id
into one warp, so that statistics keyed without the element index would differ.  The fixtures and the statistics rule defined here are the
ones the GPU suite uses.  No GPU needed."""
import numpy as np
import pytest
from scipy.ndimage import gaussian_filter

ELASTIC_BOUND = 1e-12        # max |field - scipy| / max |scipy| per field
OLD_ELASTIC_BOUND = 1e-5     # the bound the elastic field was first tested at


# ------------------------------------------------------------------------------------------------------------------ elastic field
def gauss_weights(sigma, dtype=np.float64):
    """mdt_augment_gaussian's weights: exp(k x x) with k = -0.5 / sigma^2 over [-r, r], r = int(4 sigma + 0.5), over their sequential fp64
    sum; dtype rounds the normalised weights (fp32 models a kernel that keeps them in single precision)"""
    r = int(4.0 * sigma + 0.5)
    k = -0.5 / (sigma * sigma)
    x = np.arange(-r, r + 1, dtype=np.float64)
    w = np.exp(k * x * x)
    s = 0.0
    for v in w:
        s += v
    return (w / s).astype(dtype).astype(np.float64), r


def gauss_emulate(x, sigma, alpha, dtype=np.float64):
    """the kernel's separable passes in its summation order: per output voxel, w[k] * x[pos + k] accumulated for k ascending over the window
    clipped to the axis (zeros beyond it add nothing), the last pass times alpha"""
    w, r = gauss_weights(sigma, dtype)
    y = x
    for ax in range(x.ndim):
        a = np.moveaxis(y, ax, -1)
        n = a.shape[-1]
        pad = np.zeros(a.shape[:-1] + (n + 2 * r,))
        pad[..., r:r + n] = a
        acc = np.zeros(a.shape)
        for k in range(-r, r + 1):
            acc = acc + w[k + r] * pad[..., r + k:r + k + n]
        y = np.moveaxis(acc, -1, ax)
    return y * alpha


def field_ratio(got, x, sigma, alpha):
    ref = gaussian_filter(x, sigma, mode='constant', cval=0) * alpha
    return float(np.abs(got - ref).max() / np.abs(ref).max())


ELASTIC_CASES = [((288, 288), 30.0), ((288, 288), 50.0), ((40, 36, 24), 33.0)]


@pytest.mark.parametrize("shape,sigma", ELASTIC_CASES)
def test_kernel_summation_order_meets_elastic_bound(shape, sigma):
    x = np.random.RandomState(0).rand(*shape) * 2 - 1
    ratio = field_ratio(gauss_emulate(x, sigma, 700.0), x, sigma, 700.0)
    print(shape, sigma, "fp64 emulation: %.2e" % ratio)
    assert ratio <= ELASTIC_BOUND


@pytest.mark.parametrize("shape,sigma", ELASTIC_CASES)
def test_fp32_weights_fail_elastic_bound(shape, sigma):
    """a kernel with fp32 weights is caught by the bound, and was not by the first one"""
    x = np.random.RandomState(0).rand(*shape) * 2 - 1
    ratio = field_ratio(gauss_emulate(x, sigma, 700.0, np.float32), x, sigma, 700.0)
    print(shape, sigma, "fp32 weights: %.2e" % ratio)
    assert ELASTIC_BOUND < ratio <= OLD_ELASTIC_BOUND


# ------------------------------------------------------------------------------------------------------------------ seg to boxes
def stats_of(seg):
    """mdt_augment_seg_to_boxes' statistics restated: [B, 255, 7] int32 count, min y/x/z, max y/x/z per (element, id); INT_MAX / -1 for
    absent ids; z entries 0 in 2D"""
    B = seg.shape[0]
    dim = seg.ndim - 2
    st = np.zeros((B, 255, 7), dtype=np.int32)
    st[:, :, 1:4] = 0x7fffffff
    st[:, :, 4:7] = -1
    for b in range(B):
        for k in np.unique(seg[b]):
            if k == 0:
                continue
            ix = np.argwhere(seg[b, 0] == k)
            st[b, k - 1, 0] = len(ix)
            st[b, k - 1, 1:1 + dim] = ix.min(0)
            st[b, k - 1, 4:4 + dim] = ix.max(0)
            if dim == 2:
                st[b, k - 1, 3] = 0
                st[b, k - 1, 6] = 0
    return st


def _voxel_coords(P):
    c = np.stack(np.unravel_index(np.arange(int(np.prod(P))), P), 1)
    return c if len(P) == 3 else np.concatenate([c, np.zeros((len(c), 1), c.dtype)], 1)


def warp_stats(seg, with_elem=True):
    """the kernel's warp aggregation over runs of 32 linear indices: lanes grouped by key (b * 255 + id - 1, or id - 1 alone when not
    with_elem), each group's count and coordinate extremes credited to the (element, id) of its lowest lane"""
    B = seg.shape[0]
    P = seg.shape[2:]
    pvol = int(np.prod(P))
    coords = _voxel_coords(P)
    flat = seg.reshape(-1).astype(np.int64)
    st = np.zeros((B, 255, 7), dtype=np.int64)
    st[:, :, 1:4] = 0x7fffffff
    st[:, :, 4:7] = -1
    for t0 in range(0, flat.size, 32):
        t = np.arange(t0, min(t0 + 32, flat.size))
        b, ids = t // pvol, flat[t]
        c = coords[t - b * pvol]
        keys = np.where(ids > 0, (b * 255 if with_elem else 0) + ids - 1, -1)
        for key in np.unique(keys[keys >= 0]):
            lanes = keys == key
            lead = np.argmax(lanes)
            s = st[b[lead], ids[lead] - 1]
            s[0] += lanes.sum()
            s[1:4] = np.minimum(s[1:4], c[lanes].min(0))
            s[4:7] = np.maximum(s[4:7], c[lanes].max(0))
    return st.astype(np.int32)


def straddling_runs(seg):
    """runs of 32 linear indices (warps) that hold foreground of two elements carrying the same id"""
    pvol = int(np.prod(seg.shape[2:]))
    flat = seg.reshape(-1)
    n = 0
    for t0 in range(0, flat.size, 32):
        t = np.arange(t0, min(t0 + 32, flat.size))
        b = t // pvol
        if b[0] == b[-1]:
            continue
        ids = flat[t]
        shared = set(ids[(b == b[0]) & (ids > 0)].tolist()) & set(ids[(b != b[0]) & (ids > 0)].tolist())
        n += bool(shared)
    return n


def elements_per_run(seg):
    pvol = int(np.prod(seg.shape[2:]))
    t0 = np.arange(0, seg.size, 32)
    return (np.minimum(t0 + 31, seg.size - 1) // pvol) - t0 // pvol + 1


def _class_targets(rs, seg, n_ct=None):
    return [[int(c) for c in rs.randint(0, 2, size=(n_ct or int(seg[b].max())))] if seg[b].any() else [] for b in range(seg.shape[0])]


def box_cases():
    """name -> (dim, seg [B, 1, *P] uint8, class_target)"""
    rs = np.random.RandomState(17)
    cases = {}

    def random_ids(name, B, P, n_ids, empty=()):
        seg = (rs.randint(1, n_ids + 1, size=(B, 1) + P) * (rs.rand(B, 1, *P) < 0.6)).astype(np.uint8)
        for b in range(B - 1):                           # the last voxel of an element and the first of the next carry the same id
            seg[b].reshape(-1)[-1] = seg[b + 1].reshape(-1)[0] = 1 + b % n_ids
        for b in empty:
            seg[b] = 0
        cases[name] = (len(P), seg, _class_targets(rs, seg))

    # patch volumes that are not a multiple of 32, so that warps straddle elements; ids from a small set, so that neighbours share them
    random_ids('7x9', 5, (7, 9), 3, empty=(2,))
    random_ids('33x31', 3, (33, 31), 5)
    random_ids('5x7x3', 6, (5, 7, 3), 3, empty=(4,))
    random_ids('33x31x9', 2, (33, 31, 9), 6)
    random_ids('3x5', 7, (3, 5), 2)                     # 15 voxels: one warp covers parts of three elements
    random_ids('b64', 64, (6, 5), 4, empty=(0, 63))
    # every id 1..255 (8 voxels each, 8 background) in element 0, random ids over the whole range in element 1
    P = (16, 16, 8)
    seg = np.zeros((2, 1) + P, dtype=np.uint8)
    seg[0, 0].reshape(-1)[rs.permutation(2048)[:2040]] = np.repeat(np.arange(1, 256), 8)
    seg[1, 0] = rs.randint(1, 256, size=P) * (rs.rand(*P) < 0.5)
    cases['all_ids'] = (3, seg, _class_targets(rs, seg, 255))
    # 32 distinct ids in every warp (32 singleton groups)
    P = (32, 24)
    seg = np.stack([(np.arange(768) % 32 + 1 + 32 * b).reshape(P) for b in range(2)])[:, None].astype(np.uint8)
    cases['distinct'] = (2, seg, _class_targets(rs, seg))
    # all foreground, one id per element (one group of 32 in every warp)
    seg = np.zeros((2, 1, 40, 36), dtype=np.uint8)
    seg[0], seg[1] = 7, 255
    cases['all_fg'] = (2, seg, _class_targets(rs, seg))
    return cases


STRADDLING = ['7x9', '33x31', '5x7x3', '33x31x9', '3x5', 'b64']


@pytest.mark.parametrize("name", sorted(box_cases()))
def test_warp_aggregation_with_element_key_equals_stats(name):
    dim, seg, ct = box_cases()[name]
    assert np.array_equal(warp_stats(seg), stats_of(seg))
    assert all(len(c) >= int(seg[b].max()) for b, c in enumerate(ct))


@pytest.mark.parametrize("name", STRADDLING)
def test_straddling_fixtures_catch_a_key_without_the_element(name):
    """warps span two elements that carry the same id, and statistics keyed by the id alone differ from the rule"""
    dim, seg, _ = box_cases()[name]
    assert int(np.prod(seg.shape[2:])) % 32 != 0
    assert straddling_runs(seg) > 0
    assert not np.array_equal(warp_stats(seg, with_elem=False), stats_of(seg))
    if name == '3x5':
        assert elements_per_run(seg).max() == 3


def test_id_pattern_fixtures():
    cases = box_cases()
    seg = cases['all_ids'][1]
    assert np.array_equal(np.unique(seg[0]), np.arange(256)) and len(cases['all_ids'][2][0]) == 255
    seg = cases['distinct'][1].reshape(-1, 32).astype(np.int64)
    assert all(len(np.unique(r)) == 32 for r in seg)
    seg = cases['all_fg'][1].reshape(-1, 32)
    assert (seg > 0).all() and all(len(np.unique(r)) == 1 for r in seg)
