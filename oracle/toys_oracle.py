"""numpy restatement of the toy experiment's image generator (experiments/toy_exp/generate_toys.py: multi_processing_create_image) for one
image drawn from np.random.RandomState(key), with the pixel loops replaced by vectorised disc masks.

The reference draws from numpy's global state; seeded with np.random.seed(key) first it gives exactly the arrays image() returns."""
import io
import hashlib

import numpy as np

SIDE = 320
HOLE_RADIUS = 4      # the reference's whole_diameter, used as a radius


def margin_of(class_diameters):
    """generate_experiment's foreground_margin"""
    return int(np.max(class_diameters) // 2)


def image(key, mode, class_diameters, margin=None):
    """(out float64 [2, 320, 320] (image, seg), (center_x, center_y, class_id)) of one image; margin defaults to the experiment's"""
    margin = margin_of(class_diameters) if margin is None else margin
    rs = np.random.RandomState(key)
    img = rs.rand(SIDE, SIDE)
    cx = rs.randint(margin, SIDE - margin)
    cy = rs.randint(margin, SIDE - margin)
    class_id = rs.randint(0, 2)
    y, x = np.mgrid[:SIDE, :SIDE]
    d2 = (x - cx) ** 2 + (y - cy) ** 2
    r = int(class_diameters[class_id])
    disc = d2 - r ** 2 < 0
    seg = disc.astype(np.uint8)
    img[disc] += 0.2
    if 'donuts' in mode and class_id == 1:
        hole = d2 - HOLE_RADIUS ** 2 < 0
        img[hole] -= 0.2
        if mode == 'donuts_shape':
            seg[hole] = 0
    return np.concatenate((img[None], seg[None])), (cx, cy, class_id)


def npy_bytes(arr):
    """the bytes np.save writes for arr"""
    buf = io.BytesIO()
    np.save(buf, arr)
    return buf.getvalue()


def npy_sha256(arr):
    return hashlib.sha256(npy_bytes(arr)).hexdigest()
