"""The toolkit's plots with the call surface of the reference's plotting.py: plot_batch_prediction, TrainingPlot_2Panel,
plot_prediction_hist and plot_stat_curves, written as PNG files under the reference's names.

Each function does two things.  First it builds, on the host, the figure's content with the reference's choices: which element, slices,
boxes, colours, strings, positions and series (`*_calls`, in the form of the matplotlib calls the reference makes, so tests can compare them
with the reference's recorded calls).  Then a layout step maps the content to integer pixels in fp64, once, and csrc/render.cu draws it
on the GPU: image panels (grey or class colours, nearest-neighbour up-scaling by an integer factor) and primitives (segments, dashed
polylines, alpha rectangles, glyphs of a 6 x 8 bitmap font).  The canvas is the reference figure at 100 dpi.  The PNG is written on the
host (RGB8, filter 0, zlib level PNG_ZLIB_LEVEL).

The pictures are not pixel-identical to matplotlib's (no anti-aliasing, a bitmap font, this module's own tick and legend placement); the
content is the reference's.  matplotlib is not used.  There is no CPU fallback: without a CUDA device the calls raise, like the other
native ops.
"""
import ctypes
import os
import struct
import zlib
from copy import deepcopy

import numpy as np
import torch

from . import _lib as L

DPI = 100
PNG_ZLIB_LEVEL = 1            # plots are large flat areas plus noisy image slices; level 1 compresses the first as well and is far faster
GLYPH_W, GLYPH_H = 6, 8
BASELINE = 7                  # font rows above the baseline
SEGMENT, RECT, GLYPH = 0, 1, 2
GREY, CLASS = 0, 1
DTYPE_CODE = {torch.uint8: 0, torch.float16: 1, torch.float32: 2}

# the matplotlib colour names the reference's configs and plotting.py use
COLORS = {'b': (0, 0, 255), 'c': (0, 191, 191), 'r': (255, 0, 0), 'g': (0, 128, 0), 'm': (191, 0, 191), 'y': (191, 191, 0),
          'k': (0, 0, 0), 'w': (255, 255, 255), 'purple': (128, 0, 128), 'tab:gray': (127, 127, 127)}
# matplotlib's default line colour cycle (tab10), used by the stat curves which set no colour
CYCLE = [(31, 119, 180), (255, 127, 14), (44, 160, 44), (214, 39, 40), (148, 103, 189), (140, 86, 75), (227, 119, 194), (127, 127, 127),
         (188, 189, 34), (23, 190, 207)]
# viridis at 0, 1/8, ..., 1: the class colours with vmin = 0, vmax = n - 1 are viridis(k / (n - 1)), interpolated between these
_VIRIDIS = np.array([(0x44, 0x01, 0x54), (0x47, 0x2D, 0x7B), (0x3B, 0x52, 0x8B), (0x2C, 0x72, 0x8E), (0x21, 0x91, 0x8C), (0x28, 0xAE, 0x80),
                     (0x5E, 0xC9, 0x62), (0xAD, 0xDC, 0x30), (0xFD, 0xE7, 0x25)], dtype=np.float64)
BLACK, WHITE, GRID = (0, 0, 0), (255, 255, 255), (176, 176, 176)
# the reference's default_configs.py values for what cf may lack
CF_DEFAULTS = {'box_color_palette': {'det': 'b', 'gt': 'r', 'neg_class': 'purple', 'prop': 'w', 'pos_class': 'g', 'pos_anchor': 'c',
                                     'neg_anchor': 'c'},
               'n_monitoring_figures': 1, 'assign_values_to_extra_figure': {}, 'do_validation': True, 'num_epochs': 100}
# matplotlib's default subplot parameters, and the dash pattern of linestyle '--' at linewidth 1.5 (3.7 on, 1.6 off, in linewidths)
SUBPLOT = dict(left=0.125, right=0.9, bottom=0.11, top=0.88)
DASH_ON, DASH_PERIOD = 8, 11
HIST_ALPHA = 77               # round(0.3 * 256)


def _cf_get(cf, name):
    if hasattr(cf, name):
        return getattr(cf, name)
    if name == 'plot_dir':                                  # exp_utils.prepare_monitoring's choice
        return os.path.join(cf.exp_dir, 'plots')
    return deepcopy(CF_DEFAULTS[name])


def color(name):
    """RGB of a colour name of COLORS, '#rrggbb', or an RGB tuple"""
    if isinstance(name, str):
        if name.startswith('#'):
            return tuple(int(name[i:i + 2], 16) for i in (1, 3, 5))
        return COLORS[name]
    return tuple(int(v) for v in name)


def class_palette(n):
    """uint8 [n, 3]: viridis(k / (n - 1)) for the classes k of a map drawn with vmin = 0, vmax = n - 1"""
    n = max(int(n), 1)
    t = np.arange(n, dtype=np.float64) / max(n - 1, 1) * (len(_VIRIDIS) - 1)
    i = np.minimum(np.floor(t).astype(np.int64), len(_VIRIDIS) - 2)
    f = (t - i)[:, None]
    return np.floor(_VIRIDIS[i] * (1 - f) + _VIRIDIS[i + 1] * f + 0.5).astype(np.uint8)


def glyph_scale(fontsize):
    """the integer glyph scale of a font size in points at 100 dpi (an 8-pixel cell per scale step): 7 -> 1, 10 -> 2, 20 -> 3"""
    return max(1, int(np.floor(fontsize * DPI / 72.0 / GLYPH_H + 0.5)))


def png_name(name):
    """matplotlib's savefig naming: a name without an extension gets '.png'; another extension than .png is not supported"""
    ext = os.path.splitext(name)[1]
    if ext == '':
        return name + '.png'
    if ext.lower() != '.png':
        raise ValueError('only PNG output is supported, not %r' % ext)
    return name


# ------------------------------------------------------------------------------------------------------------------------------- PNG
def encode_png(rgb):
    """bytes of an RGB8 PNG of rgb (uint8 [H, W, 3]): one IDAT, filter type 0 on every row, zlib level PNG_ZLIB_LEVEL"""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, _ = rgb.shape
    raw = np.zeros((h, 1 + 3 * w), dtype=np.uint8)
    raw[:, 1:] = rgb.reshape(h, 3 * w)

    def chunk(tag, data):
        return struct.pack('>I', len(data)) + tag + data + struct.pack('>I', zlib.crc32(tag + data) & 0xffffffff)

    return (b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, 2, 0, 0, 0))
            + chunk(b'IDAT', zlib.compress(raw.tobytes(), PNG_ZLIB_LEVEL)) + chunk(b'IEND', b''))


def write_png(path, rgb):
    with open(path, 'wb') as f:
        f.write(encode_png(rgb))


# ------------------------------------------------------------------------------------------------------------------------- the scene
class Scene:
    """a canvas size, image panels and a primitive list in integer pixels"""

    def __init__(self, width, height):
        self.width, self.height = int(width), int(height)
        self.panels = []          # (source 2-D array or tensor, y0, x0, scale, mode)
        self.prims = []           # 12-int rows of struct mdt_render_prim
        self.n_classes = 1

    def panel(self, src, y0, x0, scale, mode):
        self.panels.append((src, int(y0), int(x0), int(scale), mode))

    def segment(self, x0, y0, x1, y1, rgb, dash=None):
        on, period, offset = dash if dash is not None else (0, 0, 0)
        self.prims.append((SEGMENT, x0, y0, x1, y1, _pack(rgb), 0, 0, 0, on, period, offset))

    def polyline(self, xs, ys, rgb, dashed=False):
        """consecutive segments; a dashed polyline carries the dash phase across its joints.  Non-finite points break the line."""
        offset = 0
        for k in range(len(xs) - 1):
            if not (np.isfinite(xs[k]) and np.isfinite(ys[k]) and np.isfinite(xs[k + 1]) and np.isfinite(ys[k + 1])):
                offset = 0
                continue
            x0, y0, x1, y1 = int(xs[k]), int(ys[k]), int(xs[k + 1]), int(ys[k + 1])
            self.segment(x0, y0, x1, y1, rgb, (DASH_ON, DASH_PERIOD, offset) if dashed else None)
            offset = (offset + max(abs(x1 - x0), abs(y1 - y0))) % DASH_PERIOD

    def rect(self, x0, y0, x1, y1, rgb, alpha=256):
        self.prims.append((RECT, x0, y0, x1, y1, _pack(rgb), alpha, 0, 0, 0, 0, 0))

    def text(self, x, y, s, rgb, scale, ha='left', va='baseline'):
        """s at pixel (x, y): ha left / center / right of the advance, va baseline / top / center of the cell"""
        s = str(s)
        w = GLYPH_W * scale * len(s)
        x = x - (w // 2 if ha == 'center' else w if ha == 'right' else 0)
        top = y - BASELINE * scale if va == 'baseline' else y if va == 'top' else y - GLYPH_H * scale // 2
        for i, ch in enumerate(s):
            code = ord(ch)
            if 33 <= code <= 126:
                self.prims.append((GLYPH, x + i * GLYPH_W * scale, top, 0, 0, _pack(rgb), 0, code, scale, 0, 0, 0))
        return w

    def render(self):
        """the canvas as numpy uint8 [H, W, 3], drawn on the current CUDA device"""
        return render(self).cpu().numpy()


def _pack(rgb):
    r, g, b = color(rgb)
    return (r << 16) | (g << 8) | b


class PanelDesc(ctypes.Structure):
    """mirror of struct mdt_render_panel (include/mdt_b200.h)"""
    _fields_ = [('src', ctypes.c_void_p), ('stride_y', ctypes.c_longlong), ('stride_x', ctypes.c_longlong)] + \
               [(n, ctypes.c_int) for n in ('dtype', 'h', 'w', 'y0', 'x0', 'scale', 'mode', 'pad')]


def _device():
    if not torch.cuda.is_available():
        raise L.MdtError("plotting renders on CUDA only (there is no CPU fallback) and no CUDA device is available")
    return torch.device('cuda', torch.cuda.current_device())


def _as_source(src, dev):
    """a 2-D CUDA tensor view of dtype uint8 / fp16 / fp32; host arrays are uploaded, other dtypes converted by torch"""
    t = src if isinstance(src, torch.Tensor) else torch.from_numpy(np.asarray(src))
    if t.dtype not in DTYPE_CODE:
        t = t.to(torch.float32)
    return t.to(dev)


def _upload(rows, dev):
    buf = bytes(rows) if not isinstance(rows, np.ndarray) else rows.tobytes()
    return torch.frombuffer(bytearray(buf), dtype=torch.uint8).to(dev)


def panels_overlap(panels):
    """True when two panels' destination rectangles intersect (their pixels would be written by concurrent CTAs)"""
    if len(panels) < 2:
        return False
    r = np.array([(y0, x0, y0 + int(src.shape[0]) * s, x0 + int(src.shape[1]) * s) for src, y0, x0, s, _ in panels], dtype=np.int64)
    inter = ((np.maximum(r[:, None, 0], r[None, :, 0]) < np.minimum(r[:, None, 2], r[None, :, 2]))
             & (np.maximum(r[:, None, 1], r[None, :, 1]) < np.minimum(r[:, None, 3], r[None, :, 3])))
    np.fill_diagonal(inter, False)
    return bool(inter.any())


def render(scene):
    """the scene drawn into a white device canvas uint8 [H, W, 3] by mdt_render_panel_range, mdt_render_panels and mdt_render_prims"""
    if panels_overlap(scene.panels):
        raise ValueError('the panels of a scene must not overlap')
    dev = _device()
    lib = L.load()
    stream = L.stream_ptr()
    canvas = torch.full((scene.height, scene.width, 3), 255, dtype=torch.uint8, device=dev)
    keep = []
    if scene.panels:
        descs = (PanelDesc * len(scene.panels))()
        for d, (src, y0, x0, s, mode) in zip(descs, scene.panels):
            t = _as_source(src, dev)
            keep.append(t)
            d.src, d.stride_y, d.stride_x = t.data_ptr(), t.stride(0), t.stride(1)
            d.dtype, d.h, d.w, d.y0, d.x0, d.scale, d.mode = DTYPE_CODE[t.dtype], t.shape[0], t.shape[1], y0, x0, s, mode
        dd = _upload(descs, dev)
        rng = torch.empty((len(scene.panels), 2), dtype=torch.float32, device=dev)
        pal = torch.from_numpy(class_palette(scene.n_classes)).to(dev)
        keep += [dd, rng, pal]
        L.check(lib.mdt_render_panel_range(L.ptr(dd), len(scene.panels), L.ptr(rng), stream))
        L.check(lib.mdt_render_panels(L.ptr(dd), len(scene.panels), L.ptr(rng), L.ptr(pal), pal.shape[0], L.ptr(canvas), scene.height,
                                      scene.width, stream))
    if scene.prims:
        pr = _upload(np.asarray(scene.prims, dtype=np.int32), dev)
        keep.append(pr)
        L.check(lib.mdt_render_prims(L.ptr(pr), len(scene.prims), L.ptr(canvas), scene.height, scene.width, stream))
    torch.cuda.current_stream().synchronize()
    return canvas


# ------------------------------------------------------------------------------------------------------------ plot_batch_prediction
class _Slice:
    """a lazily taken 2-D slice of a batch array (numpy or tensor): arr[lead, ch] (2D) or arr[lead, ch, :, :, z] (3D)"""

    def __init__(self, arr, lead, ch, z=None):
        self.arr, self.lead, self.ch, self.z = arr, lead, ch, z

    def get(self):
        return self.arr[self.lead, self.ch] if self.z is None else self.arr[self.lead, self.ch, :, :, self.z]

    def numpy(self):
        v = self.get()
        v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        return v.astype(float)


def _shape(a):
    return tuple(a.shape)


def batch_prediction_calls(batch, results_dict, cf, outfile=None):
    """the reference's plot_batch_prediction content: (outfile, figsize, gridspec shape, calls), calls a list of
    ('subplot', (m, b)), ('axis', 'off'), ('title', s, {'fontsize': 20}), ('imshow', _Slice, kwargs), ('plot', xs, ys, kwargs),
    ('text', x, y, s, kwargs) in the reference's order.  Draws np.random.choice for a 3D batch, as the reference does."""
    if outfile is None:
        outfile = os.path.join(_cf_get(cf, 'plot_dir'), 'pred_example_{}.png'.format(cf.fold))
    data, segs, pids = batch['data'], batch['seg'], batch['pid']
    if len(set(pids)) == 1:
        pids = [pids] * data.shape[0]
    seg_preds = results_dict['seg_preds']
    roi_results = deepcopy(results_dict['boxes'])
    n_ch, n_seg, n_pred = data.shape[1], segs.shape[1], seg_preds.shape[1]
    if cf.dim == 3:
        patient_ix = np.random.choice(data.shape[0])
        n_z = data.shape[-1]
        gt_boxes = [box['box_coords'] for box in roi_results[patient_ix] if box['box_type'] == 'gt']
        if len(gt_boxes) > 0:
            z_cuts = [np.max((int(gt_boxes[0][4]) - 5, 0)), np.min((int(gt_boxes[0][5]) + 5, n_z))]
        else:
            z_cuts = [n_z // 2 - 5, int(n_z // 2 + np.min([10, n_z // 2]))]
        p_roi_results = roi_results[patient_ix]
        roi_results = [[] for _ in range(n_z)]
        for box in p_roi_results:
            b = box['box_coords']
            slices = np.round(np.unique(np.clip(np.arange(b[4], b[5] + 1), 0, n_z - 1)))
            for s in slices:
                roi_results[int(s)].append(box)
                roi_results[int(s)][-1]['box_coords'] = b[:4]
        zs = list(range(n_z))[z_cuts[0]:z_cuts[1]]
        roi_results = roi_results[z_cuts[0]:z_cuts[1]]
        pids = [pids[patient_ix]] * len(zs)
        shapes = [(len(zs), a.shape[1], a.shape[2], a.shape[3]) for a in (data, segs, seg_preds)]

        def cell(arr, ch, b):
            return _Slice(arr, patient_ix, ch, zs[b])
    else:
        zs = list(range(data.shape[0]))
        shapes = [_shape(a) for a in (data, segs, seg_preds)]

        def cell(arr, ch, b):
            return _Slice(arr, b, ch)
    if not all(shapes[0][i] == shapes[1][i] == shapes[2][i] for i in (0, 2, 3)):
        raise Warning('Shapes of arrays to plot not in agreement!'
                      'Shapes {} vs. {} vs {}'.format(*shapes))
    rows = [(data, c) for c in range(n_ch)] + [(segs, c) for c in range(n_seg)] + [(seg_preds, c) for c in range(n_pred)] + [(data, 0)]
    n_b, n_rows = len(zs), len(rows)
    palette = _cf_get(cf, 'box_color_palette')
    calls = []
    for b in range(n_b):
        for m in range(n_rows):
            calls += [('subplot', (m, b)), ('axis', 'off')]
            if m < n_ch or m == n_rows - 1:
                kw = {'cmap': 'gray', 'vmin': None, 'vmax': None}
            else:
                kw = {'cmap': None, 'vmin': 0, 'vmax': cf.num_seg_classes - 1}
            if m == 0:
                calls.append(('title', '{}'.format(pids[b][:10]), {'fontsize': 20}))
            calls.append(('imshow', cell(rows[m][0], rows[m][1], b), kw))
            if m < n_ch:
                continue
            for box in roi_results[b]:
                if box['box_type'] == 'patient_tn_box':
                    continue
                coords = box['box_coords']
                if box['box_type'] == 'det':
                    if not (box['box_pred_class_id'] > 0 and box['box_score'] > 0.1):
                        continue
                    plot_text = True
                    score = np.max(box['box_score'])
                    score_text = '{}|{:.0f}'.format(box['box_pred_class_id'], score * 100)
                    if 'sample_id' in box.keys() and int(box['sample_id']) != m - n_ch - 2:
                        continue
                    if 'sample_id' not in box.keys() and m != n_ch + 1:
                        continue
                    text_color, text_x, text_y = 'w', coords[1] + 10 * (box['box_pred_class_id'] - 1), coords[2] + 5
                elif box['box_type'] == 'gt':
                    plot_text = True
                    score_text = int(box['box_label'])
                    text_color, text_x, text_y = 'r', coords[1], coords[0] - 1
                else:
                    plot_text = False
                color_var = 'extra_usage' if 'extra_usage' in list(box.keys()) else 'box_type'
                kw = {'color': palette[box[color_var]], 'linewidth': 1, 'alpha': 1}
                calls += [('plot', [coords[1], coords[3]], [coords[0], coords[0]], kw), ('plot', [coords[1], coords[3]], [coords[2], coords[2]], kw),
                          ('plot', [coords[1], coords[1]], [coords[0], coords[2]], kw), ('plot', [coords[3], coords[3]], [coords[0], coords[2]], kw)]
                if plot_text:
                    calls.append(('text', text_x, text_y, score_text, {'fontsize': 7, 'color': text_color}))
    figsize = (4 * n_b, 4 * n_rows)
    return outfile, figsize, (n_rows + 1, n_b), calls


def _grid_cells(fig_w, fig_h, n_rows, n_cols, space=0.1):
    """fp64 pixel boxes (x, y, w, h), y downwards, of GridSpec(n_rows, n_cols) with wspace = hspace = space under the default subplot
    parameters"""
    cw = (SUBPLOT['right'] - SUBPLOT['left']) * fig_w / (n_cols + space * (n_cols - 1))
    ch = (SUBPLOT['top'] - SUBPLOT['bottom']) * fig_h / (n_rows + space * (n_rows - 1))
    x0, y0 = SUBPLOT['left'] * fig_w, (1 - SUBPLOT['top']) * fig_h
    return lambda r, c: (x0 + c * cw * (1 + space), y0 + r * ch * (1 + space), cw, ch)


def _round(v):
    return int(np.floor(v + 0.5))


def _device_views(slices):
    """{id(_Slice): 2-D CUDA view}: a host array goes to the device once, as the slab the figure shows (the drawn element's slices of a 3D
    batch, the whole of a 2D one); dtypes other than uint8 / fp16 / fp32 are converted on that slab"""
    dev = _device()
    slabs, views = {}, {}
    for sl in slices:
        key = id(sl.arr)
        if key not in slabs:
            if sl.z is None:
                slabs[key] = (_as_source(sl.arr, dev), 0)
            else:
                zs = [o.z for o in slices if o.arr is sl.arr]
                slabs[key] = (_as_source(sl.arr[sl.lead][..., min(zs):max(zs) + 1], dev), min(zs))
        t, z_lo = slabs[key]
        views[id(sl)] = t[sl.lead, sl.ch] if sl.z is None else t[sl.ch, :, :, sl.z - z_lo]
    return views


def batch_prediction_scene(outfile, figsize, grid, calls, n_classes):
    W, H = figsize[0] * DPI, figsize[1] * DPI
    views = _device_views([c[1] for c in calls if c[0] == 'imshow'])
    scene = Scene(W, H)
    scene.n_classes = n_classes
    cells = _grid_cells(W, H, grid[0], grid[1])
    cur = None
    place = None
    pending_title = None
    for call in calls:
        kind = call[0]
        if kind == 'subplot':
            cur = cells(*call[1])
        elif kind == 'title':
            pending_title = call[1:]
        elif kind == 'imshow':
            src = views[id(call[1])]
            h, w = int(src.shape[0]), int(src.shape[1])
            s = int(np.floor(min(cur[2] / w, cur[3] / h)))
            if s >= 1:
                dh, dw, scale = h * s, w * s, float(s)
            else:                                      # larger than its cell: every k-th pixel, a strided view
                k = int(np.ceil(max(w / cur[2], h / cur[3])))
                src, s, scale = src[::k, ::k], 1, 1.0 / k
                dh, dw = int(src.shape[0]), int(src.shape[1])
            x0, y0 = _round(cur[0] + (cur[2] - dw) / 2), _round(cur[1] + (cur[3] - dh) / 2)
            scene.panel(src, y0, x0, s, GREY if call[2]['cmap'] == 'gray' else CLASS)
            place = (x0, y0, scale)
            if pending_title is not None:
                scene.text(x0 + dw // 2, y0 - 8, pending_title[0], BLACK, glyph_scale(pending_title[1]['fontsize']), ha='center')
                pending_title = None
        elif kind in ('plot', 'text'):
            x0, y0, s = place

            def px(v):
                return int(np.floor(x0 + (float(v) + 0.5) * s))

            def py(v):
                return int(np.floor(y0 + (float(v) + 0.5) * s))
            if kind == 'plot':
                scene.polyline([px(v) for v in call[1]], [py(v) for v in call[2]], call[3]['color'])
            else:
                scene.text(px(call[1]), py(call[2]), call[3], call[4]['color'], glyph_scale(call[4]['fontsize']))
    return scene


def plot_batch_prediction(batch, results_dict, cf, outfile=None):
    """the input slices, ground-truth and predicted label maps, GT boxes (with labels) and detections (with class|score) of a batch, or of
    one randomly drawn element (np.random.choice) of a 3D batch around its first GT box; written to outfile (default
    {plot_dir}/pred_example_{fold}.png).  batch['data'], batch['seg'] and results_dict['seg_preds'] may be numpy arrays or CUDA tensors."""
    outfile, figsize, grid, calls = batch_prediction_calls(batch, results_dict, cf, outfile)
    write_png(png_name(outfile), batch_prediction_scene(outfile, figsize, grid, calls, cf.num_seg_classes).render())


# -------------------------------------------------------------------------------------------------------------------------- charts
def nice_ticks(lo, hi, max_ticks=8):
    """ticks k * step inside [lo, hi] with step 1, 2 or 5 times a power of ten, the smallest giving at most max_ticks"""
    span = hi - lo
    if not np.isfinite(span) or span <= 0:
        return np.array([lo])
    base = 10.0 ** np.floor(np.log10(span / max_ticks))
    for m in (1, 2, 5, 10, 20):
        step = m * base
        first, last = np.ceil(lo / step - 1e-9), np.floor(hi / step + 1e-9)
        if last - first + 1 <= max_ticks:
            return np.arange(first, last + 1) * step
    return np.array([lo, hi])


def _tick_label(v, step):
    if abs(v) < step * 1e-6:
        v = 0.0
    digits = max(0, -int(np.floor(np.log10(step) + 1e-9))) if step > 0 else 0
    return '{:.{}f}'.format(v, digits)


def _auto_limits(vals, log=False):
    v = np.asarray([x for x in vals if x is not None], dtype=np.float64)
    v = v[np.isfinite(v) & ((v > 0) if log else True)]
    if v.size == 0:
        return (1.0, 10.0) if log else (0.0, 1.0)
    lo, hi = v.min(), v.max()
    if log:
        lo, hi = np.log10(lo), np.log10(hi)
    if hi == lo:
        lo, hi = lo - 0.5, hi + 0.5
    pad = 0.05 * (hi - lo)
    lo, hi = lo - pad, hi + pad
    return (10 ** lo, 10 ** hi) if log else (lo, hi)


class _Chart:
    """one axes of a chart figure: limits, the data-to-pixel map (fp64, once per point) and the frame, ticks, labels and legend"""

    def __init__(self, scene, box, xlim, ylim, ylog=False):
        self.scene, self.ylog = scene, ylog
        self.x0, self.y0, self.w, self.h = box
        self.xlim, self.ylim = xlim, ylim

    def px(self, x):
        return int(np.floor(self.x0 + (float(x) - self.xlim[0]) / (self.xlim[1] - self.xlim[0]) * self.w))

    def py(self, y):
        y = float(y)
        if self.ylog:
            if not y > 0:
                return self.y0 + self.h
            t = (np.log10(y) - np.log10(self.ylim[0])) / (np.log10(self.ylim[1]) - np.log10(self.ylim[0]))
        else:
            t = (y - self.ylim[0]) / (self.ylim[1] - self.ylim[0])
        return int(np.floor(self.y0 + (1 - t) * self.h))

    def line(self, xs, ys, rgb, dashed=False):
        xp = [self.px(x) if x is not None and np.isfinite(float(x)) else np.nan for x in xs]
        yp = [self.py(y) if y is not None and np.isfinite(float(y)) else np.nan for y in ys]
        self.scene.polyline(xp, yp, rgb, dashed)

    def axes(self, grid=False, title=None, xlabel=None, ylabel=None):
        s, x0, y0, x1, y1 = self.scene, self.x0, self.y0, self.x0 + self.w, self.y0 + self.h
        if self.ylog:
            e0, e1 = int(np.ceil(np.log10(self.ylim[0]) - 1e-9)), int(np.floor(np.log10(self.ylim[1]) + 1e-9))
            yt = [(10.0 ** e, '10^%d' % e) for e in range(e0, e1 + 1)]
        else:
            t = nice_ticks(*self.ylim)
            yt = [(v, _tick_label(v, t[1] - t[0] if len(t) > 1 else 1)) for v in t]
        t = nice_ticks(*self.xlim)
        xt = [(v, _tick_label(v, t[1] - t[0] if len(t) > 1 else 1)) for v in t]
        for v, lab in xt:
            p = self.px(v)
            if grid:
                s.segment(p, y0, p, y1, GRID)
            s.segment(p, y1, p, y1 + 4, BLACK)
            s.text(p, y1 + 7, lab, BLACK, 2, ha='center', va='top')
        for v, lab in yt:
            p = self.py(v)
            if grid:
                s.segment(x0, p, x1, p, GRID)
            s.segment(x0 - 4, p, x0, p, BLACK)
            s.text(x0 - 7, p, lab, BLACK, 2, ha='right', va='center')
        for a, b, c, d in ((x0, y0, x1, y0), (x0, y1, x1, y1), (x0, y0, x0, y1), (x1, y0, x1, y1)):
            s.segment(a, b, c, d, BLACK)
        if title is not None:                         # scale 1 when scale 2 would run past the canvas
            ts = 2 if GLYPH_W * 2 * len(str(title)) <= s.width else 1
            s.text(x0 + self.w // 2, y0 - 8, title, BLACK, ts, ha='center')
        if xlabel is not None:
            s.text(x0 + self.w // 2, y1 + 30, xlabel, BLACK, 2, ha='center', va='top')
        if ylabel is not None:                        # upright glyphs, stacked top to bottom
            n = len(ylabel)
            top = y0 + self.h // 2 - n * GLYPH_H * 2 // 2
            for i, ch in enumerate(ylabel):
                s.text(max(x0 - 70, 2), top + i * GLYPH_H * 2, ch, BLACK, 2, va='top')

    def legend(self, entries, loc):
        """entries [(label, rgb, 'line' | 'dashed' | 'patch')]; loc 'upper right', 'lower left', 'lower right' or 'outside right'"""
        if not entries:
            return
        s = self.scene
        x1, y1 = self.x0 + self.w, self.y0 + self.h
        pad, sample = 8, 28
        for ts in (2, 1):                             # scale 1 when scale 2 would run past the canvas
            w = pad * 3 + sample + max(len(e[0]) for e in entries) * GLYPH_W * ts
            if (x1 + 10 if loc == 'outside right' else self.x0) + w <= s.width:
                break
        row = GLYPH_H * ts + 4
        h = pad * 2 + row * len(entries)
        if loc == 'outside right':
            lx, ly = x1 + 10, self.y0 + (self.h - h) // 2
        else:
            lx = self.x0 + pad if 'left' in loc else x1 - pad - w
            ly = self.y0 + pad if 'upper' in loc else y1 - pad - h
        s.rect(lx, ly, lx + w, ly + h, WHITE, 205)
        for a, b, c, d in ((lx, ly, lx + w, ly), (lx, ly + h, lx + w, ly + h), (lx, ly, lx, ly + h), (lx + w, ly, lx + w, ly + h)):
            s.segment(a, b, c, d, (204, 204, 204))
        for i, (label, rgb, style) in enumerate(entries):
            cy = ly + pad + i * row + row // 2
            if style == 'patch':
                s.rect(lx + pad, cy - 5, lx + pad + sample, cy + 5, rgb, HIST_ALPHA)
            else:
                s.segment(lx + pad, cy, lx + pad + sample, cy, rgb, (DASH_ON, DASH_PERIOD, 0) if style == 'dashed' else None)
            s.text(lx + 2 * pad + sample, cy, label, BLACK, ts, va='center')


def _axes_box(W, H, position=None):
    x, y, w, h = position if position is not None else (SUBPLOT['left'], SUBPLOT['bottom'], SUBPLOT['right'] - SUBPLOT['left'],
                                                        SUBPLOT['top'] - SUBPLOT['bottom'])
    return _round(x * W), _round((1 - y - h) * H), _round(w * W), _round(h * H)


# ----------------------------------------------------------------------------------------------------------- plot_prediction_hist
def prediction_hist_calls(label_list, pred_list, type_list, outfile):
    """the reference's plot_prediction_hist content: (outfile, figsize, calls)"""
    preds = np.array(pred_list)
    labels = np.array(label_list)
    title = outfile.split('/')[-1] + ' count:{}'.format(len(label_list))
    calls = [('yscale', 'log')]
    if 0 in labels:
        calls.append(('hist', preds[labels == 0], {'alpha': 0.3, 'color': 'g', 'range': (0, 1), 'bins': 50, 'label': 'false pos.'}))
    if 1 in labels:
        calls.append(('hist', preds[labels == 1], {'alpha': 0.3, 'color': 'b', 'range': (0, 1), 'bins': 50,
                                                    'label': 'true pos. (false neg. @ score=0)'}))
    if type_list is not None:
        fp_count = type_list.count('det_fp')
        fn_count = type_list.count('det_fn')
        tp_count = type_list.count('det_tp')
        title += ' tp:{} fp:{} fn:{} pos:{}'.format(tp_count, fp_count, fn_count, fn_count + tp_count)
    calls += [('legend', {}), ('title', title, {}), ('xlabel', 'confidence score'), ('ylabel', 'log n')]
    return outfile, (6.4, 4.8), calls


def prediction_hist_scene(figsize, calls):
    W, H = _round(figsize[0] * DPI), _round(figsize[1] * DPI)
    scene = Scene(W, H)
    hists = [(np.histogram(np.asarray(c[1], dtype=np.float64), bins=c[2]['bins'], range=c[2]['range'])[0], c[2]) for c in calls if c[0] == 'hist']
    counts = [v for h, _ in hists for v in h.tolist()]
    ch = _Chart(scene, _axes_box(W, H), (-0.05, 1.05), _auto_limits(counts, log=True), ylog=True)
    edges = np.linspace(0, 1, 51)
    for h, kw in hists:
        for k, n in enumerate(h):
            if n > 0:
                scene.rect(ch.px(edges[k]), ch.py(n), max(ch.px(edges[k + 1]), ch.px(edges[k]) + 1), ch.y0 + ch.h, kw['color'], HIST_ALPHA)
    d = {c[0]: c for c in calls}
    ch.axes(title=d['title'][1], xlabel=d['xlabel'][1], ylabel=d['ylabel'][1])
    ch.legend([(kw['label'], kw['color'], 'patch') for _, kw in hists], 'upper right')
    return scene


def plot_prediction_hist(label_list, pred_list, type_list, outfile):
    """log-count histograms (50 bins over [0, 1]) of the scores of the false (label 0) and true (label 1) predictions, with the counts of
    type_list in the title; written to outfile (+ '.png' without an extension)"""
    outfile, figsize, calls = prediction_hist_calls(label_list, pred_list, type_list, outfile)
    write_png(png_name(outfile), prediction_hist_scene(figsize, calls).render())


# --------------------------------------------------------------------------------------------------------------- plot_stat_curves
def stat_curves_calls(stats, outfile):
    """the reference's plot_stat_curves content: [(outfile, figsize, calls)] for 'roc' and 'prc'.  A curve that is not a tuple (the np.nan
    of a patient-level stat whose class has one label value) is skipped; the reference raises on it."""
    figs = []
    for c in ['roc', 'prc']:
        calls = []
        for s in stats:
            curve = s.get(c)
            if isinstance(curve, (tuple, list)):
                calls.append(('plot', np.asarray(curve[0]), np.asarray(curve[1]), {'label': s['name'] + '_' + c}))
        calls += [('title', outfile.split('/')[-1] + '_' + c, {}), ('legend', {'loc': 3 if c == 'prc' else 4}),
                  ('xlabel', 'precision' if c == 'prc' else '1-spec.'), ('ylabel', 'recall')]
        figs.append((outfile + '_' + c, (6.4, 4.8), calls))
    return figs


def stat_curves_scene(figsize, calls):
    W, H = _round(figsize[0] * DPI), _round(figsize[1] * DPI)
    scene = Scene(W, H)
    lines = [c for c in calls if c[0] == 'plot']
    xlim = _auto_limits([v for c in lines for v in c[1].tolist()])
    ylim = _auto_limits([v for c in lines for v in c[2].tolist()])
    ch = _Chart(scene, _axes_box(W, H), xlim, ylim)
    for k, c in enumerate(lines):
        ch.line(c[1].tolist(), c[2].tolist(), CYCLE[k % len(CYCLE)])
    d = {c[0]: c for c in calls}
    ch.axes(title=d['title'][1], xlabel=d['xlabel'][1], ylabel=d['ylabel'][1])
    ch.legend([(c[3]['label'], CYCLE[k % len(CYCLE)], 'line') for k, c in enumerate(lines)],
              'lower left' if d['legend'][1]['loc'] == 3 else 'lower right')
    return scene


def plot_stat_curves(stats, outfile):
    """ROC and PR curves of the stats with a curve, written to outfile + '_roc' and outfile + '_prc' (+ '.png')"""
    for name, figsize, calls in stat_curves_calls(stats, outfile):
        write_png(png_name(name), stat_curves_scene(figsize, calls).render())


# ------------------------------------------------------------------------------------------------------------ TrainingPlot_2Panel
class TrainingPlot_2Panel():
    """the training monitor: per figure, the train (dashed) and validation (solid) curves of the monitored values over epochs, written to
    {plot_dir}/monitor_{fold}_{figure_ix}.png by update_and_save(metrics, epoch)"""

    def __init__(self, cf):
        self.file_name = _cf_get(cf, 'plot_dir') + '/monitor_{}'.format(cf.fold)
        self.exp_name = cf.fold_dir
        self.do_validation = _cf_get(cf, 'do_validation')
        self.separate_values_dict = _cf_get(cf, 'assign_values_to_extra_figure')
        self.figure_calls = []
        for n in range(_cf_get(cf, 'n_monitoring_figures')):
            self.figure_calls.append([('subplot', 111), ('xlabel', 'epochs'), ('ylabel', 'loss / metrics'), ('xlim', 0, _cf_get(cf, 'num_epochs')),
                                      ('grid',)])
        self.figure_calls[0].append(('ylim', 0, 1.5))
        self.color_palette = ['b', 'c', 'r', 'purple', 'm', 'y', 'k', 'tab:gray']
        self.figsize = (10, 6)

    def update_calls(self, metrics, epoch):
        """appends this epoch's calls to every figure; returns [(file name, figsize, calls so far)], one per figure"""
        out = []
        for figure_ix in range(len(self.figure_calls)):
            calls = self.figure_calls[figure_ix]
            calls += monitoring_calls(metrics, self.exp_name, self.color_palette, epoch, figure_ix, self.separate_values_dict,
                                      self.do_validation)
            out.append((self.file_name + '_{}'.format(figure_ix), self.figsize, list(calls)))
        return out

    def update_and_save(self, metrics, epoch):
        for name, figsize, calls in self.update_calls(metrics, epoch):
            write_png(png_name(name), monitor_scene(figsize, calls).render())


def monitoring_calls(metrics, exp_name, color_palette, epoch, figure_ix, separate_values_dict, do_validation):
    """the calls of the reference's detection_monitoring_plot for one figure and epoch"""
    monitor_values_keys = metrics['train']['monitor_values'][1][0].keys()
    separate_values = [v for fig_ix in separate_values_dict.values() for v in fig_ix]
    if figure_ix == 0:
        plot_keys = [ii for ii in monitor_values_keys if ii not in separate_values]
        plot_keys += [k for k in metrics['train'].keys() if k != 'monitor_values']
    else:
        plot_keys = separate_values_dict[figure_ix]
    x = np.arange(1, epoch + 1)
    calls = []
    for kix, pk in enumerate(plot_keys):
        if pk in metrics['train'].keys():
            y_train = metrics['train'][pk][1:]
            if do_validation:
                y_val = metrics['val'][pk][1:]
        else:
            y_train = [np.mean([er[pk] for er in metrics['train']['monitor_values'][e]]) for e in x]
            if do_validation:
                y_val = [np.mean([er[pk] for er in metrics['val']['monitor_values'][e]]) for e in x]
        calls.append(('plot', x, list(y_train), {'label': 'train_{}'.format(pk), 'linestyle': '--', 'color': color_palette[kix]}))
        if do_validation:
            calls.append(('plot', x, list(y_val), {'label': 'val_{}'.format(pk), 'linestyle': '-', 'color': color_palette[kix]}))
    if epoch == 1:
        pos = (SUBPLOT['left'], SUBPLOT['bottom'], SUBPLOT['right'] - SUBPLOT['left'], SUBPLOT['top'] - SUBPLOT['bottom'])
        calls += [('set_position', [pos[0], pos[1], pos[2] * 0.8, pos[3]]), ('legend', {'loc': 'center left', 'bbox_to_anchor': (1, 0.5)}),
                  ('title', exp_name, {})]
    return calls


def monitor_scene(figsize, calls):
    """the monitor figure.  Each epoch re-plots every curve over the previous epochs' shorter copies with the same style and data, so only
    the last epoch's lines are drawn; the legend lists the lines present when legend() was called, as matplotlib does."""
    W, H = _round(figsize[0] * DPI), _round(figsize[1] * DPI)
    scene = Scene(W, H)
    d, position, legend_at = {}, None, None
    for i, c in enumerate(calls):
        if c[0] == 'set_position':
            position = c[1]
        elif c[0] == 'legend':
            legend_at = i
        elif c[0] in ('xlabel', 'ylabel', 'title', 'xlim', 'ylim'):
            d[c[0]] = c
    plots = [(i, c) for i, c in enumerate(calls) if c[0] == 'plot']
    last = {}
    for i, c in plots:                                 # the latest call per label
        last[c[3]['label']] = (i, c)
    lines = [c for i, c in sorted(last.values(), key=lambda t: t[0])]
    xlim = (d['xlim'][1], d['xlim'][2]) if 'xlim' in d else _auto_limits([v for c in lines for v in c[1]])
    ylim = (d['ylim'][1], d['ylim'][2]) if 'ylim' in d else _auto_limits([v for c in lines for v in c[2]])
    ch = _Chart(scene, _axes_box(W, H, position), xlim, ylim)
    ch.axes(grid=True, title=d['title'][1] if 'title' in d else None, xlabel=d['xlabel'][1], ylabel=d['ylabel'][1])
    for c in lines:
        ch.line(c[1], c[2], c[3]['color'], dashed=c[3]['linestyle'] == '--')
    if legend_at is not None:
        seen = []
        for i, c in plots:
            if i < legend_at and c[3]['label'] not in [s[0] for s in seen]:
                seen.append((c[3]['label'], c[3]['color'], 'dashed' if c[3]['linestyle'] == '--' else 'line'))
        ch.legend(seen, 'outside right')
    return scene
