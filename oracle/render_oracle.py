"""numpy rasteriser of csrc/render.cu's scene: the same integer rules and the same fp32 grey mapping, one primitive at a time in list order.
It is the reference the GPU tests compare the kernels against bit for bit.  The font is read from render.cu's table, so both draw the same
glyphs.

Panels are dicts {'src': 2-D numpy array (float32, float16 or uint8), 'y0', 'x0', 'scale', 'mode'}; primitives are an int32 [n, 12] array
with the fields of struct mdt_render_prim (include/mdt_b200.h) in order."""
import os
import re

import numpy as np

GREY, CLASS = 0, 1
SEGMENT, RECT, GLYPH = 0, 1, 2
GLYPH_W, GLYPH_H = 6, 8
COORD_LIMIT = 1 << 24
(KIND, X0, Y0, X1, Y1, RGB, ALPHA, CODE, SCALE, DASH_ON, DASH_PERIOD, DASH_OFFSET) = range(12)

_RENDER_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'medicaldetectiontoolkit_b200', 'csrc', 'render.cu')
_font = None


def font():
    """uint8 [95, 8]: the rows of codes 32 .. 126, bit 5 the leftmost column (render.cu's c_font)"""
    global _font
    if _font is None:
        text = open(_RENDER_CU).read()
        body = text[text.index('c_font[95]'):]
        body = body[body.index('{') + 1:body.index('};')]
        vals = [int(v, 16) for v in re.findall(r'0x([0-9a-fA-F]{2})', body)]
        assert len(vals) == 95 * GLYPH_H
        _font = np.array(vals, dtype=np.uint8).reshape(95, GLYPH_H)
    return _font


def panel_range(src):
    """(lo, hi) as fp32 over the finite values; (0, 0) without one"""
    v = np.asarray(src).astype(np.float32)
    v = v[np.isfinite(v)]
    if v.size == 0:
        return np.float32(0), np.float32(0)
    return v.min(), v.max()


def draw_panels(canvas, panels, palette=None):
    H, W, _ = canvas.shape
    for p in panels:
        src = np.asarray(p['src']).astype(np.float32)
        s = int(p['scale'])
        if src.ndim != 2 or src.size == 0 or s < 1:
            continue
        lo, hi = panel_range(src)
        if p['mode'] == GREY:
            if hi > lo:
                with np.errstate(invalid='ignore'):
                    t = (src - lo) / np.float32(hi - lo)
                    g = np.minimum(255, np.nan_to_num(t * np.float32(256), nan=0, posinf=0, neginf=0).astype(np.int64))
            else:
                g = np.zeros(src.shape, np.int64)
            rgb = np.repeat(g[..., None], 3, axis=2).astype(np.uint8)
        else:
            pal = np.asarray(palette, dtype=np.uint8).reshape(-1, 3)
            k = np.clip(np.nan_to_num(src, nan=0, posinf=0, neginf=0), 0, pal.shape[0] - 1).astype(np.int64)
            rgb = pal[k]
        finite = np.isfinite(src)
        big = np.repeat(np.repeat(rgb, s, axis=0), s, axis=1)
        fin = np.repeat(np.repeat(finite, s, axis=0), s, axis=1)
        y0, x0 = int(p['y0']), int(p['x0'])
        ya, yb = max(y0, 0), min(y0 + big.shape[0], H)
        xa, xb = max(x0, 0), min(x0 + big.shape[1], W)
        if ya >= yb or xa >= xb:
            continue
        sub = (slice(ya - y0, yb - y0), slice(xa - x0, xb - x0))
        dst = canvas[ya:yb, xa:xb]
        m = fin[sub]
        dst[m] = big[sub][m]
    return canvas


def _bbox(q):
    if any(abs(int(q[i])) > COORD_LIMIT for i in (X0, Y0, X1, Y1)):
        return None
    k = q[KIND]
    if k == SEGMENT:
        if q[DASH_PERIOD] < 0 or (q[DASH_PERIOD] > 0 and (q[DASH_ON] <= 0 or q[DASH_OFFSET] < 0)):
            return None
        return min(q[X0], q[X1]), min(q[Y0], q[Y1]), max(q[X0], q[X1]), max(q[Y0], q[Y1])
    if k == RECT:
        if not 0 <= q[ALPHA] <= 256 or q[X0] >= q[X1] or q[Y0] >= q[Y1]:
            return None
        return q[X0], q[Y0], q[X1] - 1, q[Y1] - 1
    if k == GLYPH:
        if not 33 <= q[CODE] <= 126 or not 1 <= q[SCALE] <= COORD_LIMIT:
            return None
        return q[X0], q[Y0], q[X0] + GLYPH_W * q[SCALE] - 1, q[Y0] + GLYPH_H * q[SCALE] - 1
    return None


def segment_mask(q, px, py):
    """the pixels (px, py) (int64 arrays) that segment q covers, by the closed form of render.cu's on_segment"""
    x0, y0, x1, y1 = (int(q[i]) for i in (X0, Y0, X1, Y1))
    dx, dy = x1 - x0, y1 - y0
    adx, ady = abs(dx), abs(dy)
    if adx == 0 and ady == 0:
        on = (px == x0) & (py == y0)
        t = np.zeros_like(px)
    elif adx >= ady:
        t = px - x0 if dx > 0 else x0 - px
        off = (2 * ady * t + adx) // (2 * adx)
        on = (t >= 0) & (t <= adx) & (py == y0 + (-off if dy < 0 else off))
    else:
        t = py - y0 if dy > 0 else y0 - py
        off = (2 * adx * t + ady) // (2 * ady)
        on = (t >= 0) & (t <= ady) & (px == x0 + (-off if dx < 0 else off))
    if q[DASH_PERIOD] > 0:
        on &= ((int(q[DASH_OFFSET]) + t) % int(q[DASH_PERIOD])) < int(q[DASH_ON])
    return on


def draw_prims(canvas, prims):
    H, W, _ = canvas.shape
    f = font()
    for q in np.asarray(prims, dtype=np.int64).reshape(-1, 12):
        bb = _bbox(q)
        if bb is None:
            continue
        xa, ya, xb, yb = max(bb[0], 0), max(bb[1], 0), min(bb[2], W - 1), min(bb[3], H - 1)
        if xa > xb or ya > yb:
            continue
        py, px = np.mgrid[ya:yb + 1, xa:xb + 1].astype(np.int64)
        col = np.array([(q[RGB] >> 16) & 255, (q[RGB] >> 8) & 255, q[RGB] & 255], dtype=np.int64)
        dst = canvas[ya:yb + 1, xa:xb + 1]
        if q[KIND] == SEGMENT:
            dst[segment_mask(q, px, py)] = col
        elif q[KIND] == RECT:
            a = int(q[ALPHA])
            dst[...] = ((a * col + (256 - a) * dst.astype(np.int64) + 128) >> 8).astype(np.uint8)
        else:
            s = int(q[SCALE])
            cx, cy = (px - q[X0]) // s, (py - q[Y0]) // s
            on = (f[q[CODE] - 32][cy] >> (GLYPH_W - 1 - cx)) & 1
            dst[on.astype(bool)] = col
    return canvas


def render(canvas, panels, prims, palette=None):
    """canvas uint8 [H, W, 3] (modified in place and returned): the panels, then the primitives"""
    draw_panels(canvas, panels, palette)
    return draw_prims(canvas, prims)
