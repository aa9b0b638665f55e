"""Times plotting.py at sizes users run: plot_batch_prediction of a lidc 3D validation batch (8 x 128 x 128 x 64, 20 slices drawn) and of a
2D batch (20 x 288 x 288), and plot_prediction_hist of 96 000 rows.

Per figure: the render kernels' device time (CUDA events around mdt_render_panel_range + mdt_render_panels + mdt_render_prims, inputs
already on the device), the device-to-host copy of the canvas, the PNG encoding, the whole public call (host arrays in, file out), and the
numpy oracle's rendering of the same scene on one host core.  Prints one JSON line per figure, with the card, its power limit and max SM
clock read in the same run.

    python tools/plot_bench.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import render_oracle as R  # noqa: E402

from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import plotting as P  # noqa: E402


class CF:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def batch(dim, B, shape, seed):
    rs = np.random.RandomState(seed)
    data = rs.randn(B, 1, *shape).astype(np.float32)
    seg = np.zeros((B, 1) + shape, np.uint8)
    seg_preds = np.zeros((B, 1) + shape, np.int64)
    boxes = []
    for b in range(B):
        bl = []
        for k in range(3):
            y, x = rs.randint(10, shape[0] - 40), rs.randint(10, shape[1] - 40)
            c = [y, x, y + 20, x + 24] + ([20 + 4 * k, 30 + 4 * k] if dim == 3 else [])
            seg[(b, 0, slice(y, y + 20), slice(x, x + 24))] = 1
            seg_preds[(b, 0, slice(y + 2, y + 22), slice(x + 1, x + 25))] = 1
            bl.append({'box_coords': np.array(c, np.float64), 'box_type': 'gt', 'box_label': 1 + k % 2})
            bl.append({'box_coords': np.array(c, np.float64) + 2, 'box_type': 'det', 'box_score': 0.5 + 0.1 * k, 'box_pred_class_id': 1 + k % 2})
        for k in range(30):
            y, x = rs.randint(0, shape[0] - 20), rs.randint(0, shape[1] - 20)
            c = [y, x, y + 16, x + 16] + ([rs.randint(0, shape[2] - 8)] * 2 if dim == 3 else [])
            bl.append({'box_coords': np.array(c, np.float64), 'box_type': 'pos_anchor' if k % 2 else 'neg_anchor'})
        boxes.append(bl)
    return ({'data': data, 'seg': seg, 'pid': ['p%d' % b for b in range(B)]}, {'boxes': boxes, 'seg_preds': seg_preds},
            CF(dim=dim, num_seg_classes=3, fold=0))


def kernel_ms(scene, reps):
    """device time of the three entry points on inputs already on the device"""
    lib, stream, dev = L.load(), L.stream_ptr(), torch.device('cuda')
    canvas = torch.full((scene.height, scene.width, 3), 255, dtype=torch.uint8, device=dev)
    srcs = [P._as_source(src, dev) for src, *_ in scene.panels]
    descs = (P.PanelDesc * max(len(srcs), 1))()
    for d, t, (_, y0, x0, s, mode) in zip(descs, srcs, scene.panels):
        d.src, d.stride_y, d.stride_x = t.data_ptr(), t.stride(0), t.stride(1)
        d.dtype, d.h, d.w, d.y0, d.x0, d.scale, d.mode = P.DTYPE_CODE[t.dtype], t.shape[0], t.shape[1], y0, x0, s, mode
    dd = P._upload(descs, dev)
    rng = torch.empty((max(len(srcs), 1), 2), dtype=torch.float32, device=dev)
    pal = torch.from_numpy(P.class_palette(scene.n_classes)).to(dev)
    pr = P._upload(np.asarray(scene.prims, dtype=np.int32), dev) if scene.prims else None

    def run():
        if srcs:
            L.check(lib.mdt_render_panel_range(L.ptr(dd), len(srcs), L.ptr(rng), stream))
            L.check(lib.mdt_render_panels(L.ptr(dd), len(srcs), L.ptr(rng), L.ptr(pal), pal.shape[0], L.ptr(canvas), scene.height, scene.width,
                                          stream))
        if pr is not None:
            L.check(lib.mdt_render_prims(L.ptr(pr), len(scene.prims), L.ptr(canvas), scene.height, scene.width, stream))
    run()                                             # one pass from white is the picture; the timed passes redraw over it
    rgb = canvas.cpu().numpy()
    for _ in range(2):
        run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        run()
    b.record()
    b.synchronize()
    t_d2h = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        canvas.cpu()
        t_d2h.append(time.perf_counter() - t0)
    return a.elapsed_time(b) / reps, 1e3 * float(np.median(t_d2h)), rgb


def measure(name, build_scene, public_call, reps):
    scene = build_scene()
    k_ms, d2h_ms, rgb = kernel_ms(scene, reps)
    t_png = []
    for _ in range(3):
        t0 = time.perf_counter()
        png = P.encode_png(rgb)
        t_png.append(time.perf_counter() - t0)
    t_call = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        public_call()
        t_call.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    init = np.full((scene.height, scene.width, 3), 255, np.uint8)
    want = R.render(init, [{'src': P._as_source(s, 'cpu').float().numpy(), 'y0': y0, 'x0': x0, 'scale': sc, 'mode': m}
                           for s, y0, x0, sc, m in scene.panels], np.asarray(scene.prims, np.int32).reshape(-1, 12), P.class_palette(scene.n_classes))
    t_oracle = time.perf_counter() - t0
    return {'figure': name, 'canvas': [scene.width, scene.height], 'panels': len(scene.panels), 'prims': len(scene.prims),
            'kernels_ms': round(k_ms, 3), 'd2h_ms': round(d2h_ms, 2), 'png_ms': round(1e3 * float(np.median(t_png)), 1), 'png_bytes': len(png),
            'call_ms': round(1e3 * float(np.median(t_call)), 1), 'oracle_ms': round(1e3 * t_oracle, 1), 'equal_oracle': bool(np.array_equal(rgb, want))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None, help='directory for the PNG files (default: a temporary directory)')
    args = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip().splitlines()
    card = card[0] if card else torch.cuda.get_device_name()
    out = args.out or tempfile.mkdtemp(prefix='plot_bench_')
    os.makedirs(out, exist_ok=True)
    torch.cuda.init()
    for name, dim, B, shape in (('lidc_3d', 3, 8, (128, 128, 64)), ('batch_2d', 2, 20, (288, 288))):
        b, res, cf = batch(dim, B, shape, 0)
        path = os.path.join(out, 'pred_example_%s.png' % name)

        def build():
            np.random.seed(0)
            o, fs, grid, calls = P.batch_prediction_calls(b, res, cf, path)
            return P.batch_prediction_scene(o, fs, grid, calls, cf.num_seg_classes)

        def call():
            np.random.seed(0)
            P.plot_batch_prediction(b, res, cf, path)
        print(json.dumps(dict(measure(name, build, call, args.reps), card=card)), flush=True)
    rs = np.random.RandomState(1)
    labels = (rs.rand(96000) < 0.1).astype(int).tolist()
    preds = rs.rand(96000).tolist()
    types_ = ['det_tp' if l else 'det_fp' for l in labels]
    hist = os.path.join(out, 'pred_hist_0_val_rois_cl1')

    def build_hist():
        _, fs, calls = P.prediction_hist_calls(labels, preds, types_, hist)
        return P.prediction_hist_scene(fs, calls)
    print(json.dumps(dict(measure('hist_96k', build_hist, lambda: P.plot_prediction_hist(labels, preds, types_, hist), args.reps), card=card)),
          flush=True)


if __name__ == '__main__':
    main()
