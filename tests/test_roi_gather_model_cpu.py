"""Executable statement of why the RoIAlign backward gather may cull RoIs by the taps of their end bins (csrc/roi_align.cu:
axis_meets_tile in roi_bwd_gather): along each axis, the sampling coordinate of bin o is monotone in o (every step of sample_coord - a product
of o by the scale, FMAs, a rounding to float, a clamp to [0, size - 1] - is monotone, increasing for hi >= lo and decreasing for inverted
boxes), so floor and ceil are too and every bin's taps lie between those of the first and the last bin.  The taps come from
tests/roi_gather_model.c, which computes them as nvcc compiles sample_coord; the inputs are adversarial for rounding (coordinates that land
on or one ulp beside a voxel centre, clamped ends, inverted and zero-extent boxes, crop extent 1, large maps).  The last test checks the
restated backward itself against an fp64 scatter."""
import numpy as np
import pytest

import _roi_gather_model as M

CROPS = [1, 2, 3, 5, 7, 14, 28, 64, 65, 100]
SIZES = [1, 2, 3, 7, 16, 31, 128, 1000, 4099]


def _check_axis(lo, hi, crop, size):
    tlo, thi, lerp = M.taps(lo, hi, crop, size)
    fmin, fmax = M.footprint(lo, hi, crop, size)
    assert fmin == tlo.min() and fmax == thi.max(), (lo, hi, crop, size, fmin, fmax, tlo, thi)   # the end bins bound every bin
    assert (tlo >= 0).all() and (thi <= size - 1).all()
    step = np.diff(tlo.astype(np.int64))
    assert (step >= 0).all() if hi >= lo else (step <= 0).all(), (lo, hi, crop, size, tlo)       # monotone in the bin index
    assert ((thi == tlo) == (lerp == 0)).all() and ((thi - tlo) <= 1).all()


def _adversarial(size, crop, rs):
    """box ends whose sample coordinates sit on, or one float step beside, a voxel centre, plus clamped, inverted and degenerate boxes"""
    f = np.float32
    ends = []
    for k in rs.randint(-2, size + 3, size=6):
        c = f(k + 0.5) / f(size)
        ends += [c, np.nextafter(c, f(np.inf)), np.nextafter(c, f(-np.inf)), f(k) / f(size)]
    ends += [f(0), f(1), f(-0.25), f(1.25), f(-1e-7), f(1 + 1e-7), f(0.5)]
    out = []
    for _ in range(60):
        a, b = rs.choice(len(ends), 2)
        out.append((ends[a], ends[b]))
    out += [(f(0.3), f(0.3)), (f(1), f(1)), (f(0), f(0)), (f(0.9), f(0.1)), (f(1.3), f(-0.4))]
    return out


def test_end_bins_bound_every_bins_taps():
    rs = np.random.RandomState(0)
    n = 0
    for size in SIZES:
        for crop in CROPS:
            boxes = [tuple(np.float32(v) for v in rs.uniform(-0.5, 1.5, size=2)) for _ in range(25)]
            for lo, hi in boxes + _adversarial(size, crop, rs):
                _check_axis(lo, hi, crop, size)
                n += 1
    assert n > 8000


def test_clamped_and_inverted_boxes_keep_their_taps_inside():
    """a box wholly past the far border samples size - 1 everywhere (lo == hi, lerp 0); one before the origin samples 0; an inverted box
    runs its taps downwards"""
    tlo, thi, lerp = M.taps(np.float32(1.2), np.float32(1.6), 7, 10)
    assert (tlo == 9).all() and (thi == 9).all() and (lerp == 0).all()
    assert M.footprint(np.float32(1.2), np.float32(1.6), 7, 10) == (9, 9)
    tlo, thi, _ = M.taps(np.float32(-0.6), np.float32(-0.1), 5, 10)
    assert (tlo == 0).all() and (thi == 0).all()
    tlo, thi, _ = M.taps(np.float32(0.9), np.float32(0.1), 7, 20)
    assert tlo[0] > tlo[-1] and M.footprint(np.float32(0.9), np.float32(0.1), 7, 20) == (int(tlo[-1]), int(thi[0]))


def test_sample_coord_contracts_like_nvcc():
    """lo * size + o * scale is one FMA in the kernels (exact product, one rounding): find inputs where that differs from rounding the product
    first, and check that the model takes the fused value there"""
    from fractions import Fraction
    f = np.float32
    rs = np.random.RandomState(1)
    found = 0
    for lo in rs.uniform(0, 1, size=2000).astype(f):
        hi, o, crop, size = f(lo + f(0.25)), 3, 7, 33
        scale = f(f(f(hi - lo) * f(size)) / f(crop))
        p = f(f(o) * scale)
        d = np.float64(lo) * np.float64(size) + np.float64(p)
        if Fraction(float(d)) != Fraction(float(lo)) * size + Fraction(float(p)):
            continue                                            # the double sum rounded: f32(d) could double-round
        fused, unfused = f(d), f(f(lo * f(size)) + p)
        if fused == unfused:
            continue
        s2 = np.float64(fused) + np.float64(scale) * 0.5        # exact in double: both terms are floats of similar magnitude
        want = min(f(np.float64(f(s2)) - 0.5), f(size - 1))
        assert M.lib().model_sample_coord(lo, hi, o, crop, size) == want, lo
        found += 1
    assert found >= 10


@pytest.mark.parametrize("dim", [2, 3])
def test_restated_backward_is_the_adjoint(dim):
    """the restated gather agrees with an fp64 scatter of the same taps to fp32 rounding, and zero_init = 0 adds to the prior content"""
    rs = np.random.RandomState(dim)
    B, C, n = 2, 3, 12
    sp = (9, 7, 5)[:dim]
    crop = (4, 3, 2)[:dim]
    lo = rs.uniform(-0.2, 0.8, size=(n, dim))
    hi = lo + rs.uniform(-0.1, 0.6, size=(n, dim))
    cols = [lo[:, 0], lo[:, 1], hi[:, 0], hi[:, 1]] + ([lo[:, 2], hi[:, 2]] if dim == 3 else [])
    boxes = np.stack(cols, 1).astype(np.float32)
    ind = rs.randint(-1, B + 1, size=n).astype(np.int32)
    g = rs.randn(n, C, *crop).astype(np.float32)
    shape = (B, C) + sp
    gs = [int(s) // 4 for s in g.strides]
    is5 = [int(s) // 4 for s in np.empty(shape, np.float32).strides]
    got = M.gather_backward(g.ravel(), gs, boxes, ind, np.zeros(int(np.prod(shape)), np.float32), is5, shape, crop, 1).reshape(shape)
    ref = np.zeros(shape)
    ax = []
    for a in range(dim):
        c0, c1 = (4, 5) if a == 2 else (a, a + 2)
        ax.append([M.taps(boxes[i, c0], boxes[i, c1], crop[a], sp[a]) for i in range(n)])
    for i in range(n):
        if not 0 <= ind[i] < B:
            continue
        for o in np.ndindex(*crop):
            for k in np.ndindex(*(2,) * dim):
                w, idx = 1.0, []
                for a in range(dim):
                    tlo, thi, lerp = ax[a][i]
                    w *= float(lerp[o[a]]) if k[a] else 1.0 - float(lerp[o[a]])
                    idx.append(int(thi[o[a]] if k[a] else tlo[o[a]]))
                ref[(ind[i], slice(None)) + tuple(idx)] += w * g[(i, slice(None)) + o].astype(np.float64)
    assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()
    assert (got[:, :, ...] != 0).any()
    prior = rs.randn(*shape).astype(np.float32)
    again = M.gather_backward(g.ravel(), gs, boxes, ind, prior.ravel().copy(), is5, shape, crop, 0).reshape(shape)
    assert np.abs(again - (prior + ref)).max() <= 1e-5 * np.abs(prior + ref).max()
