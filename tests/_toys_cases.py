"""The toy-generator cases shared by the golden script and the tests, and a numpy stand-in for generate_toys.CudaOps.

A case is one experiment directory: `n` images in each split, image `six` of split `s` (0 = train, 1 = test) drawn from
np.random.RandomState([seed, s, six])."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
import toys_oracle as TO  # noqa: E402

SPLITS = ('train', 'test')

# name, mode, class_diameters, seed, images per split
CASES = [
    ('donuts_shape', 'donuts_shape', (20, 20), 0, 6),
    ('donuts_pattern', 'donuts_pattern', (20, 20), 8, 6),
    ('circles_scale', 'circles_scale', (19, 20), 2, 6),
    ('donuts_shape_noise', 'donuts_shape_noise', (20, 20), 3, 6),
    ('circles', 'circles', (20, 20), 4, 6),
    ('shape_5_30', 'donuts_shape', (5, 30), 5, 6),        # margin 15, discs of radius 30 cut by the border
    ('shape_3_3', 'donuts_shape', (3, 3), 6, 6),          # the hole (radius 4) reaches past the disc (radius 3)
    ('pattern_0_20', 'donuts_pattern', (0, 20), 7, 6),    # class 0 has no disc
]


def keys(seed, split, n, start=0):
    return np.array([[seed, split, six] for six in range(start, start + n)], dtype=np.uint32)


class NumpyOps(object):
    """generate_toys.CudaOps on the host: the oracle's images and a plain (unpinned) staging buffer"""

    def images(self, keys, mode, class_diameters, margin):
        outs = [TO.image([int(k) for k in key], mode, class_diameters, margin) for key in keys]
        img = torch.from_numpy(np.stack([o[0] for o in outs]))
        params = torch.tensor([o[1] for o in outs], dtype=torch.int32).reshape(-1, 3)
        return img, params

    def staging(self, n):
        return torch.empty((n, 2, TO.SIDE, TO.SIDE), dtype=torch.float64)
