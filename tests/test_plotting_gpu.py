"""csrc/render.cu bit for bit against the numpy rasteriser (oracle/render_oracle.py), through guarded exact-size canvases that start from
random bytes, and plotting.py end to end: real model outputs, the evaluator's files, and byte-identical reruns."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import render_oracle as R  # noqa: E402
from _guarded import OFFSETS, _Guarded  # noqa: E402
from test_plotting_cpu import _decode  # noqa: E402

from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import plotting as P  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _dev_bytes(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(DEV)


def _panel_descs(panels):
    """panels [(tensor view on DEV, y0, x0, scale, mode)] -> device array of struct mdt_render_panel"""
    descs = (P.PanelDesc * len(panels))()
    for d, (t, y0, x0, s, mode) in zip(descs, panels):
        d.src, d.stride_y, d.stride_x = t.data_ptr(), t.stride(0), t.stride(1)
        d.dtype, d.h, d.w, d.y0, d.x0, d.scale, d.mode = P.DTYPE_CODE[t.dtype], t.shape[0], t.shape[1], y0, x0, s, mode
    return _dev_bytes(bytes(descs))


def gpu_vs_oracle(W, H, panels=(), prims=(), n_classes=3, seed=0, offsets=OFFSETS):
    """every entry point on a guarded canvas [H, W, 3] of random bytes at each base offset; each result equals the oracle's from the same
    bytes, and nothing outside the canvas is written"""
    lib = L.load()
    stream = L.stream_ptr()
    init = np.random.RandomState(seed).randint(0, 256, (H, W, 3)).astype(np.uint8)
    pal = P.class_palette(n_classes)
    want = R.render(init.copy(), [{'src': t.float().cpu().numpy(), 'y0': y0, 'x0': x0, 'scale': s, 'mode': m} for t, y0, x0, s, m in panels],
                    np.asarray(prims, dtype=np.int32).reshape(-1, 12), pal)
    pr = _dev_bytes(np.asarray(prims, dtype=np.int32).tobytes()) if len(prims) else None
    pd = _panel_descs(panels) if len(panels) else None
    dpal = torch.from_numpy(pal).to(DEV)
    for off in offsets:
        canvas = _Guarded(init.nbytes, off, 0)
        canvas.data().copy_(torch.from_numpy(init.reshape(-1)).to(DEV))
        rng = _Guarded(8 * max(len(panels), 1), off, 0xFF)
        if pd is not None:
            L.check(lib.mdt_render_panel_range(L.ptr(pd), len(panels), rng.ptr(), stream))
            L.check(lib.mdt_render_panels(L.ptr(pd), len(panels), rng.ptr(), L.ptr(dpal), n_classes, canvas.ptr(), H, W, stream))
        if pr is not None:
            L.check(lib.mdt_render_prims(L.ptr(pr), len(prims), canvas.ptr(), H, W, stream))
        torch.cuda.synchronize()
        canvas.check_guards()
        rng.check_guards()
        got = canvas.data().cpu().numpy().reshape(H, W, 3)
        if not np.array_equal(got, want):
            ys, xs = np.nonzero((got != want).any(-1))
            raise AssertionError('%d pixels differ, first at (x %d, y %d): %s vs %s' % (ys.size, xs[0], ys[0], got[ys[0], xs[0]], want[ys[0], xs[0]]))
        if panels:
            r = rng.data().view(torch.float32).cpu().numpy().reshape(-1, 2)
            for k, (t, *_rest) in enumerate(panels):
                lo, hi = R.panel_range(t.float().cpu().numpy())
                assert r[k].tolist() == [float(lo), float(hi)], k
    return want


def seg(x0, y0, x1, y1, rgb, dash=(0, 0, 0)):
    return [R.SEGMENT, x0, y0, x1, y1, rgb, 0, 0, 0] + list(dash)


def test_segments_every_octant_and_direction():
    rs = np.random.RandomState(1)
    prims = []
    for a in np.linspace(0, 2 * np.pi, 72, endpoint=False):
        for r in (1, 7, 40):
            prims.append(seg(50, 45, 50 + int(round(r * np.cos(a))), 45 + int(round(r * np.sin(a))), int(rs.randint(1 << 24))))
    prims += [seg(x, y, x, y, 0x123456) for x, y in rs.randint(0, 90, (20, 2))]                 # zero length
    prims += [seg(*rs.randint(-20, 120, 4), int(rs.randint(1 << 24))) for _ in range(100)]
    gpu_vs_oracle(101, 90, prims=prims)


def test_dashed_polylines_carry_the_phase_across_joints():
    s = P.Scene(120, 80)
    rs = np.random.RandomState(2)
    for k in range(6):
        s.polyline(rs.randint(-10, 130, 9).tolist(), rs.randint(-10, 90, 9).tolist(), P.CYCLE[k], dashed=True)
    prims = list(s.prims) + [seg(0, 5, 100, 60, 0xFF00FF, (3, 7, 5)), seg(100, 60, 0, 5, 0x00FFFF, (1, 2, 1))]
    gpu_vs_oracle(120, 80, prims=prims)


def test_primitives_off_canvas_and_straddling_every_edge():
    W, H = 70, 45
    rs = np.random.RandomState(3)
    prims = []
    for x0, y0, x1, y1 in [(-5, 10, 20, 10), (60, 20, 90, 30), (10, -8, 12, 8), (30, 40, 35, 60), (-30, -30, 100, 80), (-9, -9, -1, -1),
                           (W, 0, W + 5, 5), (0, H, 5, H + 9), (-100000, 3, 100000, 40), (1 << 24, 0, 0, 0), ((1 << 24) + 1, 0, 0, 0)]:
        prims.append(seg(x0, y0, x1, y1, int(rs.randint(1 << 24))))
        prims.append([R.RECT, x0, min(y0, y1), x1, max(y0, y1) + 1, int(rs.randint(1 << 24)), int(rs.randint(0, 257)), 0, 0, 0, 0, 0])
    for x, y in [(-3, 5), (W - 4, 10), (20, -5), (30, H - 3), (-20, -20), (W + 1, 0), (-6, 0)]:
        prims.append([R.GLYPH, x, y, 0, 0, 0xFF0000, 0, ord('W'), 1, 0, 0, 0])
        prims.append([R.GLYPH, x - 5, y - 9, 0, 0, 0x0000FF, 0, ord('#'), 3, 0, 0, 0])
    # arguments outside the ranges draw nothing
    prims += [[R.RECT, 0, 0, W, H, 0, 257, 0, 0, 0, 0, 0], [R.RECT, 0, 0, W, H, 0, -1, 0, 0, 0, 0, 0], [R.GLYPH, 0, 0, 0, 0, 0, 0, 127, 1, 0, 0, 0],
              [R.GLYPH, 0, 0, 0, 0, 0, 0, 65, 0, 0, 0, 0], [R.GLYPH, 0, 0, 0, 0, 0, 0, 32, 2, 0, 0, 0], seg(0, 0, 9, 9, 0, (0, 5, 0)),
              seg(0, 0, 9, 9, 0, (1, 5, -1)), [7, 0, 0, 9, 9, 0, 0, 0, 0, 0, 0, 0]]
    gpu_vs_oracle(W, H, prims=prims)


def test_more_primitives_than_a_chunk_stacked_alpha_and_every_glyph():
    rs = np.random.RandomState(4)
    prims = []
    for k in range(700):
        kind = k % 3
        x0, y0 = rs.randint(-10, 200), rs.randint(-10, 120)
        if kind == 0:
            prims.append(seg(x0, y0, x0 + rs.randint(-60, 60), y0 + rs.randint(-60, 60), int(rs.randint(1 << 24))))
        elif kind == 1:
            prims.append([R.RECT, x0, y0, x0 + rs.randint(1, 50), y0 + rs.randint(1, 40), int(rs.randint(1 << 24)), int(rs.randint(0, 257)), 0, 0, 0,
                          0, 0])
        else:
            prims.append([R.GLYPH, x0, y0, 0, 0, int(rs.randint(1 << 24)), 0, int(rs.randint(33, 127)), int(rs.randint(1, 4)), 0, 0, 0])
    prims += [[R.RECT, 5, 5, 60, 60, 0x2040F0, 77, 0, 0, 0, 0, 0]] * 9
    for code in range(32, 127):
        i = code - 32
        prims.append([R.GLYPH, 2 + (i % 30) * 6, 130 + (i // 30) * 8, 0, 0, 0x000000, 0, code, 1, 0, 0, 0])
        prims.append([R.GLYPH, (i % 15) * 13, 165 + (i // 15) * 17, 0, 0, 0x800000, 0, code, 2, 0, 0, 0])
    gpu_vs_oracle(197, 280, prims=prims)


def test_canvas_wider_than_65535_tiles():
    W, H = 65536 * 16 + 37, 5
    prims = [seg(0, 0, W - 1, H - 1, 0xFF0000), seg(W - 40, 0, W + 10, 4, 0x00FF00), [R.RECT, W - 20, 1, W + 3, 3, 0x0000FF, 200, 0, 0, 0, 0, 0],
             [R.GLYPH, W - 3, -2, 0, 0, 0, 0, ord('M'), 1, 0, 0, 0], seg(1048000, 0, 1048100, 4, 0x123456, (2, 3, 1))]
    gpu_vs_oracle(W, H, prims=prims, offsets=(0,))


def test_strided_panels_of_every_dtype_and_degenerate_ranges():
    rs = np.random.RandomState(5)
    base = torch.from_numpy(rs.randn(2, 3, 9, 11, 4).astype(np.float32)).to(DEV)            # [B, C, Y, X, Z]
    cl = torch.from_numpy(rs.randn(7, 13, 3).astype(np.float32)).to(DEV)                    # channels last
    u8 = torch.from_numpy(rs.randint(0, 256, (10, 12)).astype(np.uint8)).to(DEV)
    h16 = torch.from_numpy((rs.randn(8, 9) * 100).astype(np.float16)).to(DEV)
    nan = torch.full((5, 6), float('nan'), device=DEV)
    inf = torch.from_numpy(np.array([[np.inf, -np.inf, 1.0], [2.0, np.nan, 3.0]], np.float32)).to(DEV)
    only_inf = torch.from_numpy(np.array([[np.inf, -np.inf]], np.float32)).to(DEV)
    classes = torch.from_numpy(rs.randint(-2, 5, (6, 7)).astype(np.float32) + 0.5).to(DEV)
    panels = [(base[1, 2, :, :, 3], 0, 0, 3, R.GREY), (cl[:, :, 1], 0, 40, 2, R.GREY), (u8.t(), 30, 0, 2, R.GREY), (h16, 30, 30, 3, R.GREY),
              (torch.full((4, 4), 2.5, device=DEV), 60, 0, 2, R.GREY), (nan, 60, 20, 2, R.GREY), (inf, 60, 40, 4, R.GREY),
              (only_inf, 70, 70, 3, R.GREY), (classes, 80, 0, 3, R.CLASS), (u8[:6, :6], 80, 30, 2, R.CLASS),
              (base[0, 0, :, :, 0], 95, 60, 5, R.GREY)]                                     # straddles the right and bottom edges
    gpu_vs_oracle(100, 120, panels=panels, prims=[seg(0, 0, 99, 119, 0xFF0000)], n_classes=4)


def test_argument_errors():
    lib = L.load()
    s = L.stream_ptr()
    buf = torch.zeros(3 * 16 * 16, dtype=torch.uint8, device=DEV)
    assert lib.mdt_render_prims(None, -1, L.ptr(buf), 16, 16, s) == -1
    assert lib.mdt_render_prims(None, 0, L.ptr(buf), 0, 16, s) == -1
    assert lib.mdt_render_prims(None, 0, L.ptr(buf), 16 * 65536, 1, s) == -3
    assert lib.mdt_render_panels(None, 1, None, None, 0, L.ptr(buf), 16, 16, s) == -1
    assert lib.mdt_render_panel_range(None, 70000, None, s) == -1


# ---------------------------------------------------------------------------------------------------------------------- end to end
def _scene_vs_oracle(scene):
    got = scene.render()
    init = np.full((scene.height, scene.width, 3), 255, np.uint8)
    panels = [{'src': P._as_source(src, DEV).float().cpu().numpy(), 'y0': y0, 'x0': x0, 'scale': s, 'mode': m} for src, y0, x0, s, m in scene.panels]
    want = R.render(init, panels, np.asarray(scene.prims, dtype=np.int32).reshape(-1, 12), P.class_palette(scene.n_classes))
    assert np.array_equal(got, want)
    return got


def _model_case(model, dim, patch, seed):
    from medicaldetectiontoolkit_b200 import mrcnn, retina_unet
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    cf = make_cf(model, dim, patch)
    torch.manual_seed(seed)
    net = (retina_unet if model == 'retina_unet' else mrcnn).net(cf, None).to(DEV)
    batch = synthetic_batch(cf, 2, seed=seed, with_masks=model == 'mrcnn')
    with torch.no_grad():
        res = net.train_forward(batch, is_validation=True)
    return cf, batch, res


@pytest.mark.parametrize('model,dim,patch', [('retina_unet', 3, (64, 64, 32)), ('retina_unet', 2, (96, 96)), ('mrcnn', 2, (128, 128)),
                                             ('mrcnn', 3, (64, 64, 32))])
def test_batch_prediction_of_real_model_outputs(model, dim, patch, tmp_path):
    cf, batch, res = _model_case(model, dim, patch, 0)
    cf.plot_dir = str(tmp_path)
    np.random.seed(0)
    outfile, figsize, grid, calls = P.batch_prediction_calls(batch, res, cf)
    scene = P.batch_prediction_scene(outfile, figsize, grid, calls, cf.num_seg_classes)
    rgb = _scene_vs_oracle(scene)
    assert rgb.shape == (figsize[1] * 100, figsize[0] * 100, 3)
    assert any(c[0] == 'text' and c[4]['color'] == 'r' for c in calls)              # the GT boxes are labelled
    # the public call on CUDA tensors writes the same picture
    tb = dict(batch, data=torch.from_numpy(batch['data']).to(DEV), seg=torch.from_numpy(batch['seg']).to(DEV))
    tr = dict(res, seg_preds=torch.from_numpy(np.asarray(res['seg_preds'])).to(DEV))
    np.random.seed(0)
    P.plot_batch_prediction(tb, tr, cf)
    assert np.array_equal(_decode(open(os.path.join(str(tmp_path), 'pred_example_0.png'), 'rb').read()), rgb)


def test_charts_equal_the_oracle():
    rs = np.random.RandomState(6)
    labels = (rs.rand(96000) < 0.2).astype(int).tolist()
    preds = rs.rand(96000).tolist()
    _, figsize, calls = P.prediction_hist_calls(labels, preds, ['det_tp'] * 10 + ['det_fp'] * 5, '/x/pred_hist_0_val_rois_cl1')
    _scene_vs_oracle(P.prediction_hist_scene(figsize, calls))
    fpr = np.sort(rs.rand(30))
    stats = [{'name': 'a', 'roc': (fpr, np.sort(rs.rand(30)), None), 'prc': (fpr, fpr[::-1], None)}, {'name': 'b', 'roc': None, 'prc': None}]
    for _, figsize, calls in P.stat_curves_calls(stats, '/x/0_test_stat_curves'):
        _scene_vs_oracle(P.stat_curves_scene(figsize, calls))


class _CF:
    pass


def test_monitor_files(tmp_path):
    cf = _CF()
    cf.plot_dir, cf.fold, cf.fold_dir, cf.n_monitoring_figures, cf.assign_values_to_extra_figure = str(tmp_path), 0, 'fold_0', 2, {1: ['b']}
    tp = P.TrainingPlot_2Panel(cf)
    m = {k: {'monitor_values': {}, 'ap': [np.nan]} for k in ('train', 'val')}
    for e in (1, 2, 3):
        for k in m:
            m[k]['monitor_values'][e] = [{'a': 0.5 + 0.1 * e, 'b': 0.2 * e}]
            m[k]['ap'].append(0.1 * e if e != 2 else None)
        tp.update_and_save(m, e)
    assert sorted(os.listdir(str(tmp_path))) == ['monitor_0_0.png', 'monitor_0_1.png']
    for f in os.listdir(str(tmp_path)):
        assert _decode(open(os.path.join(str(tmp_path), f), 'rb').read()).shape == (600, 1000, 3)


def test_evaluator_writes_the_reference_files_only_with_a_plot_dir(tmp_path):
    import make_eval_golden as G
    from medicaldetectiontoolkit_b200 import evaluator as E
    cf, batch, res = _model_case('retina_unet', 3, (64, 64, 32), 0)
    results_list = [[res['boxes'], list(batch['pid'])]]
    cf.plot_stat_curves = True
    ev = E.Evaluator(cf, G.Logger(), 'val_sampling')
    before = set(os.listdir(str(tmp_path)))
    ev.evaluate_predictions(results_list, G.new_monitor_metrics(cf))
    cf.plot_dir = str(tmp_path / 'missing')
    ev.evaluate_predictions(results_list, G.new_monitor_metrics(cf))
    assert set(os.listdir(str(tmp_path))) == before
    cf.plot_dir = str(tmp_path)
    ev = E.Evaluator(cf, G.Logger(), 'val_sampling')
    stats, _ = ev.evaluate_predictions(results_list, G.new_monitor_metrics(cf))
    want = {'pred_hist_0_val_{}_cl{}.png'.format(level, cl) for cl in cf.class_dict for level in cf.report_score_level}
    want |= {'0_val_sampling_stat_curves_roc.png', '0_val_sampling_stat_curves_prc.png'}
    assert set(os.listdir(str(tmp_path))) == want
    for f in want:
        img = _decode(open(os.path.join(str(tmp_path), f), 'rb').read())
        assert img.shape == (480, 640, 3) and (img != 255).any()


def test_two_runs_write_byte_identical_files(tmp_path):
    cf, batch, res = _model_case('retina_unet', 3, (64, 64, 32), 1)
    out = []
    for k in range(2):
        d = tmp_path / ('run%d' % k)                  # the same file names: the histogram's title holds its name
        d.mkdir()
        np.random.seed(3)
        P.plot_batch_prediction(batch, res, cf, outfile=str(d / 'pred.png'))
        P.plot_prediction_hist([0, 1, 1, 0], [0.1, 0.5, 0.9, 0.3], None, str(d / 'hist'))
        out.append((open(str(d / 'pred.png'), 'rb').read(), open(str(d / 'hist.png'), 'rb').read()))
    assert out[0] == out[1]


def test_slices_larger_than_their_cell_are_down_sampled_without_overlap():
    """a 2D batch of 20 x 288 x 288 at 400 px per column: each slice is wider than its grid cell, drawn as every 2nd pixel"""
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import plot_bench
    b, res, cf = plot_bench.batch(2, 20, (288, 288), 0)
    np.random.seed(0)
    outfile, figsize, grid, calls = P.batch_prediction_calls(b, res, cf, 'x.png')
    scene = P.batch_prediction_scene(outfile, figsize, grid, calls, cf.num_seg_classes)
    assert not P.panels_overlap(scene.panels) and all(int(src.shape[1]) == 144 for src, *_ in scene.panels)
    _scene_vs_oracle(scene)
