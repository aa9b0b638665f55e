"""plotting.py without a GPU: the content each function builds equals the matplotlib calls the reference's plotting.py makes on the same
inputs (recorded in tests/golden/plot_calls.pkl.gz by tests/golden/make_plot_golden.py), the numpy rasteriser's rules on hand-worked cases,
and the PNG writer."""
import copy
import gzip
import os
import pickle
import struct
import sys
import zlib

import numpy as np
import pytest

from medicaldetectiontoolkit_b200 import plotting as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import render_oracle as R  # noqa: E402

GOLDEN = pickle.load(gzip.open(os.path.join(ROOT, 'tests', 'golden', 'plot_calls.pkl.gz')))


class CF:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def same(a, b, path='call'):
    if isinstance(a, P._Slice):
        a = a.numpy()
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype, path
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        A, B = np.asarray(a), np.asarray(b)
        if A.dtype == object or B.dtype == object:
            assert len(A) == len(B), path
            for i, (x, y) in enumerate(zip(A.tolist(), B.tolist())):
                same(x, y, '%s[%d]' % (path, i))
            return
        assert A.shape == B.shape and np.array_equal(A, B, equal_nan=True), path
        return
    if isinstance(a, dict):
        assert isinstance(b, dict) and sorted(a) == sorted(b), path
        for k in a:
            same(a[k], b[k], '%s.%s' % (path, k))
        return
    if isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), (path, a, b)
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, '%s[%d]' % (path, i))
        return
    if isinstance(a, float) and isinstance(b, float) and np.isnan(a) and np.isnan(b):
        return
    assert a == b and type(a) is type(b) or (isinstance(a, (int, float, np.number)) and isinstance(b, (int, float, np.number)) and a == b), \
        (path, a, b)


def same_calls(mine, ref):
    assert [c[0] for c in mine] == [c[0] for c in ref]
    for k, (x, y) in enumerate(zip(mine, ref)):
        same(x, y, 'call %d %s' % (k, x[0]))


@pytest.mark.parametrize('k', range(len(GOLDEN['batch'])))
def test_batch_prediction_content_equals_the_reference(k):
    g = GOLDEN['batch'][k]
    case = g['case']
    np.random.seed(case['seed'])
    outfile, figsize, grid, calls = P.batch_prediction_calls(copy.deepcopy(case['batch']), copy.deepcopy(case['results_dict']),
                                                             CF(**case['cf']))
    fig, = g['figures']
    assert outfile == fig['file'] and tuple(figsize) == fig['figsize']
    assert list(grid) == fig['gridspec'][:2] and fig['gridspec'][2] == {'wspace': 0.1, 'hspace': 0.1}
    same_calls(calls, fig['calls'])


def test_batch_prediction_covers_every_box_rule():
    """the fixture exercises what the filters decide: det rows, sample_id rows, dropped low-score / class-0 / tn boxes, extra_usage colours"""
    texts = [c for g in GOLDEN['batch'] for c in g['figures'][0]['calls'] if c[0] == 'text']
    plots = [c for g in GOLDEN['batch'] for c in g['figures'][0]['calls'] if c[0] == 'plot']
    assert {c[4]['color'] for c in texts} == {'w', 'r'}
    assert {c[3]['color'] for c in plots} >= {'b', 'r', 'g', 'c', 'w'}
    assert any(t[3] == '1|87' for t in texts) and not any(t[3].startswith('1|5') for t in texts if isinstance(t[3], str))


@pytest.mark.parametrize('k', range(len(GOLDEN['hist'])))
def test_prediction_hist_content_equals_the_reference(k):
    g = GOLDEN['hist'][k]
    outfile, figsize, calls = P.prediction_hist_calls(**g['case'])
    fig, = g['figures']
    assert outfile == fig['file'] and figsize == fig['figsize']
    same_calls(calls, fig['calls'])


def test_stat_curves_content_equals_the_reference():
    g = GOLDEN['stat'][0]
    figs = P.stat_curves_calls(**g['case'])
    assert len(figs) == len(g['figures']) == 2
    for (name, figsize, calls), fig in zip(figs, g['figures']):
        assert name == fig['file'] and figsize == fig['figsize']
        same_calls(calls, fig['calls'])


def test_stat_curves_skip_a_nan_curve_where_the_reference_raises():
    g = GOLDEN['stat'][1]
    assert g['raises'] == 'TypeError' and g['figures'] == []
    stats = g['case']['stats']
    with_nan = P.stat_curves_calls(stats, g['case']['outfile'])
    without = P.stat_curves_calls([s for s in stats if isinstance(s['roc'], tuple) or s['roc'] is None], g['case']['outfile'])
    for a, b in zip(with_nan, without):
        assert a[0] == b[0]
        same_calls(a[2], b[2])


@pytest.mark.parametrize('k', range(len(GOLDEN['monitor'])))
def test_monitor_content_equals_the_reference(k):
    g = GOLDEN['monitor'][k]
    tp = P.TrainingPlot_2Panel(CF(**g['case']['cf']))
    saved = []
    for e, m in g['case']['epochs']:
        saved += tp.update_calls(m, e)
    assert len(saved) == len(g['figures'])
    for (name, figsize, calls), fig in zip(saved, g['figures']):
        assert name == fig['file'] and figsize == fig['figsize']
        same_calls(calls, fig['calls'])


def test_cf_defaults_are_the_references():
    cf = CF(plot_dir='/p', fold=0, fold_dir='/f')
    tp = P.TrainingPlot_2Panel(cf)
    assert tp.do_validation is True and tp.separate_values_dict == {} and len(tp.figure_calls) == 1
    assert ('xlim', 0, 100) in tp.figure_calls[0]
    assert P._cf_get(CF(exp_dir='/e'), 'plot_dir') == os.path.join('/e', 'plots')
    assert P._cf_get(cf, 'box_color_palette')['neg_class'] == 'purple'


def test_names_colours_and_scales():
    assert P.png_name('a/b') == 'a/b.png' and P.png_name('a/b.png') == 'a/b.png'
    with pytest.raises(ValueError):
        P.png_name('a/b.pdf')
    assert [P.glyph_scale(s) for s in (7, 10, 20)] == [1, 2, 3]
    assert P.class_palette(3).tolist() == [[0x44, 0x01, 0x54], [0x21, 0x91, 0x8C], [0xFD, 0xE7, 0x25]]
    assert P.class_palette(2).tolist() == [[0x44, 0x01, 0x54], [0xFD, 0xE7, 0x25]]
    for name in ('b', 'c', 'r', 'g', 'm', 'y', 'k', 'w', 'purple', 'tab:gray'):
        assert len(P.color(name)) == 3


def test_nice_ticks():
    assert P.nice_ticks(0, 1).tolist() == pytest.approx([0, 0.2, 0.4, 0.6, 0.8, 1.0])
    assert P.nice_ticks(0, 100).tolist() == pytest.approx([0, 20, 40, 60, 80, 100])
    assert P.nice_ticks(-0.05, 1.05).tolist() == pytest.approx([0, 0.2, 0.4, 0.6, 0.8, 1.0])


def test_overlapping_panels_are_rejected():
    a = np.zeros((4, 5))
    assert not P.panels_overlap([(a, 0, 0, 2, 0), (a, 8, 0, 2, 0), (a, 0, 10, 1, 0)])
    assert P.panels_overlap([(a, 0, 0, 2, 0), (a, 7, 9, 1, 0)])
    with pytest.raises(ValueError):
        P.render(_two_panel_scene())


def _two_panel_scene():
    s = P.Scene(20, 20)
    s.panel(np.zeros((4, 4), np.float32), 0, 0, 2, 0)
    s.panel(np.zeros((4, 4), np.float32), 7, 7, 1, 0)
    return s


def test_dashes_carry_across_polyline_joints():
    s = P.Scene(100, 100)
    s.polyline([0, 5, 5, 20], [0, 0, 9, 9], 'k', dashed=True)
    offs = [p[11] for p in s.prims]
    assert offs == [0, 5, (5 + 9) % P.DASH_PERIOD]


# --------------------------------------------------------------------------------------------------------------- the oracle's rules
def _seg(x0, y0, x1, y1, on=0, period=0, offset=0):
    return [R.SEGMENT, x0, y0, x1, y1, 0x000000, 0, 0, 0, on, period, offset]


def _drawn(prims, W=12, H=10):
    c = np.full((H, W, 3), 255, np.uint8)
    R.draw_prims(c, np.array(prims))
    return sorted((int(x), int(y)) for y, x in zip(*np.nonzero(c[..., 0] == 0)))


def test_oracle_segment_closed_form():
    # x-major, slope 2/5: y = floor((2*2*t + 5) / 10)
    assert _drawn([_seg(0, 0, 5, 2)]) == [(0, 0), (1, 0), (2, 1), (3, 1), (4, 2), (5, 2)]
    # reversed ends give the mirror rounding from the other end
    assert _drawn([_seg(5, 2, 0, 0)]) == [(0, 0), (1, 0), (2, 1), (3, 1), (4, 2), (5, 2)]
    assert _drawn([_seg(3, 1, 3, 4)]) == [(3, 1), (3, 2), (3, 3), (3, 4)]
    assert _drawn([_seg(4, 4, 4, 4)]) == [(4, 4)]
    assert _drawn([_seg(0, 0, 3, 3)]) == [(0, 0), (1, 1), (2, 2), (3, 3)]
    assert _drawn([_seg(-5, 2, 2, 2)]) == [(0, 2), (1, 2), (2, 2)]


def test_oracle_dashes():
    assert _drawn([_seg(0, 0, 9, 0, on=2, period=5, offset=0)]) == [(0, 0), (1, 0), (5, 0), (6, 0)]
    assert _drawn([_seg(0, 0, 9, 0, on=2, period=5, offset=4)]) == [(1, 0), (2, 0), (6, 0), (7, 0)]


def test_oracle_alpha_and_order():
    c = np.zeros((2, 2, 3), np.uint8)
    rect = [R.RECT, 0, 0, 1, 1, 0xFF0000, 128, 0, 0, 0, 0, 0]
    R.draw_prims(c, np.array([rect, rect]))
    # (128 * 255 + 128 * 0 + 128) >> 8 = 128, then (128 * 255 + 128 * 128 + 128) >> 8 = 192
    assert c[0, 0].tolist() == [192, 0, 0] and c[1, 1].tolist() == [0, 0, 0]
    c = np.zeros((2, 2, 3), np.uint8)
    R.draw_prims(c, np.array([[R.RECT, 0, 0, 2, 2, 0x00FF00, 256, 0, 0, 0, 0, 0], _seg(0, 0, 1, 0)]))
    assert c[0, 0].tolist() == [0, 0, 0] and c[1, 0].tolist() == [0, 255, 0]


def test_oracle_glyph_and_font():
    f = R.font()
    assert f.shape == (95, 8) and not f[0].any() and (f & 1).sum() == 0     # space is blank; column 5 is the gap
    for code in range(33, 127):
        assert f[code - 32].any(), chr(code)
    c = np.full((16, 12, 3), 255, np.uint8)
    R.draw_prims(c, np.array([[R.GLYPH, 0, 0, 0, 0, 0, 0, ord('I'), 2, 0, 0, 0]]))
    on = c[..., 0] == 0
    want = np.kron(((f[ord('I') - 32][:, None] >> (5 - np.arange(6))) & 1).astype(bool), np.ones((2, 2), bool))
    assert np.array_equal(on, want)


def test_oracle_grey_mapping():
    src = np.array([[0, 1, 2, 3], [np.nan, np.inf, 4, 3.999]], np.float32)
    c = np.full((2, 4, 3), 7, np.uint8)
    R.draw_panels(c, [{'src': src, 'y0': 0, 'x0': 0, 'scale': 1, 'mode': R.GREY}])
    assert c[..., 0].tolist() == [[0, 64, 128, 192], [7, 7, 255, 255]]
    c = np.full((2, 2, 3), 7, np.uint8)
    R.draw_panels(c, [{'src': np.full((1, 1), 3.0, np.float32), 'y0': 1, 'x0': 1, 'scale': 2, 'mode': R.GREY}])
    assert c[..., 0].tolist() == [[7, 7], [7, 0]]


# ----------------------------------------------------------------------------------------------------------------------------- PNG
def _decode(png):
    assert png[:8] == b'\x89PNG\r\n\x1a\n'
    pos, chunks = 8, {}
    while pos < len(png):
        n, = struct.unpack('>I', png[pos:pos + 4])
        tag, data = png[pos + 4:pos + 8], png[pos + 8:pos + 8 + n]
        assert struct.unpack('>I', png[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + data) & 0xffffffff
        chunks[tag] = chunks.get(tag, b'') + data
        pos += 12 + n
    w, h, depth, ctype, comp, filt, inter = struct.unpack('>IIBBBBB', chunks[b'IHDR'])
    assert (depth, ctype, comp, filt, inter) == (8, 2, 0, 0, 0) and b'IEND' in chunks
    raw = np.frombuffer(zlib.decompress(chunks[b'IDAT']), np.uint8).reshape(h, 1 + 3 * w)
    assert not raw[:, 0].any()
    return raw[:, 1:].reshape(h, w, 3)


def test_png_round_trip(tmp_path):
    rgb = np.random.RandomState(0).randint(0, 256, (37, 53, 3)).astype(np.uint8)
    path = str(tmp_path / 'x.png')
    P.write_png(path, rgb)
    assert np.array_equal(_decode(open(path, 'rb').read()), rgb)
    try:
        from PIL import Image
    except ImportError:
        return
    assert np.array_equal(np.asarray(Image.open(path).convert('RGB')), rgb)
