"""Synthetic raw LIDC directories for the preprocessing tests, generated from a seed, and a numpy stand-in for preprocessing.CudaOps.

A raw file keeps the name the LIDC conversion tool gives it ({pid}_ct_scan.nrrd, {pid}_nod_{nodule id}_{roi id}.nii.gz) but holds an
.npy array; the (x, y, z) spacing of every file of a patient sits in the sidecar spacing.json of the patient's directory."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
import preprocess_oracle as PO  # noqa: E402

SEED = 20261018
TARGET_SPACING = (0.7, 0.7, 1.25)
SIDECAR = 'spacing.json'

# pid, (z, y, x), spacing (x, y, z), ROIs: (roi id, [(nodule id, malignancy, blob centre (z, y, x), radii (z, y, x))] one per rater)
PATIENTS = [
    # upsampling on every axis; ids 1 and 11 ('1.nii' selects the files of both), 1 rater and 4 raters, overlapping
    ('LIDC-IDRI-0001', (24, 40, 48), (0.9, 0.85, 2.0), [
        ('1', [(11, 4, (12, 20, 24), (4, 6, 6))]),
        ('11', [(21, 3, (13, 22, 27), (5, 6, 7)), (22, 5, (12, 22, 26), (4, 7, 7)), (23, 4, (13, 21, 27), (5, 6, 6)),
                (24, 2, (12, 23, 28), (4, 5, 7))]),
        ('2', [(31, 1, (6, 8, 10), (3, 4, 4)), (32, 2, (6, 9, 10), (3, 4, 5)), (33, 2, (7, 8, 11), (3, 4, 4))]),
    ]),
    # downsampling on every axis, gaussian radii 1 (x), 2 (y) and 3 (z); a suppressed ROI (one rater of four)
    ('LIDC-IDRI-0002', (24, 40, 48), (0.5, 0.4, 0.5), [
        ('1', [(41, 3, (12, 20, 20), (6, 8, 8)), (42, 4, (12, 21, 21), (6, 8, 9)), (43, 5, (11, 20, 20), (6, 9, 8))]),
        ('2', [(44, 2, (10, 28, 34), (5, 6, 6))]),
        ('3', [(45, 1, (14, 12, 12), (6, 7, 7)), (46, 1, (14, 12, 13), (6, 7, 7)), (47, 2, (15, 13, 12), (6, 7, 6)),
               (48, 1, (14, 11, 12), (5, 7, 7))]),
    ]),
    # mixed: x at exactly the target 0.7 (skimage's 2-D warp branch), y downsampled, z upsampled
    ('LIDC-IDRI-0003', (24, 40, 44), (0.7, 0.6, 2.0), [
        ('1', [(51, 5, (10, 18, 20), (4, 6, 6)), (52, 4, (11, 19, 21), (4, 6, 6))]),
    ]),
    # no ROI files
    ('LIDC-IDRI-0004', (20, 36, 40), (0.62, 0.62, 1.5), []),
]


def _blob(shape, centre, radii):
    z, y, x = np.ogrid[:shape[0], :shape[1], :shape[2]]
    d = sum(((g - c) / float(r)) ** 2 for g, c, r in zip((z, y, x), centre, radii))
    return (d <= 1.0).astype(np.uint8)


def roi_file(pid, nodule, rid):
    return '%s_nod_%04d_%s.nii.gz' % (pid, nodule, rid)


def ct_volume(rs, shape):
    """int16 CT-like values: air, tissue, a bright structure, noise; some values past the [-1200, 600] clip"""
    z, y, x = np.ogrid[:shape[0], :shape[1], :shape[2]]
    body = ((y - shape[1] / 2.0) / (shape[1] * 0.42)) ** 2 + ((x - shape[2] / 2.0) / (shape[2] * 0.42)) ** 2 <= 1.0
    v = np.where(body, 40.0, -1000.0) + rs.normal(0, 60, shape)
    v += np.where(rs.rand(*shape) < 0.01, 2500.0, 0.0) - np.where(rs.rand(*shape) < 0.01, 600.0, 0.0)
    return np.broadcast_to(v, shape).round().astype(np.int16)


def make_raw_dir(root):
    """writes root/characteristics.csv and root/data_nrrd/{pid}/...; returns the raw data directory"""
    rs = np.random.RandomState(SEED)
    raw = os.path.join(root, 'data_nrrd')
    rows = ['PatientID;NoduleID;Malignancy']
    for pid, shape, spacing, rois in PATIENTS:
        d = os.path.join(raw, pid)
        os.makedirs(d)
        sidecar = {}

        def put(name, arr):
            with open(os.path.join(d, name), 'wb') as f:
                np.save(f, arr)
            sidecar[name] = list(spacing)
        put('%s_ct_scan.nrrd' % pid, ct_volume(rs, shape))
        for rid, raters in rois:
            for nodule, mal, centre, radii in raters:
                put(roi_file(pid, nodule, rid), _blob(shape, centre, radii))
                rows.append('%s;%d;%d' % (pid, nodule, mal))
        with open(os.path.join(d, SIDECAR), 'w') as f:
            json.dump(sidecar, f)
    with open(os.path.join(root, 'characteristics.csv'), 'w') as f:
        f.write('\n'.join(rows) + '\n')
    return raw


def npy_reader(path):
    """read_image for the synthetic directories: (array, spacing (x, y, z))"""
    with open(os.path.join(os.path.dirname(path), SIDECAR)) as f:
        spacing = json.load(f)[os.path.basename(path)]
    return np.load(path), tuple(float(s) for s in spacing)


class NumpyOps(object):
    """numpy stand-in for preprocessing.CudaOps on preprocess_oracle; stats='numpy' normalises with numpy's float32 statistics as the
    reference does, stats='device' with the device's fp64 statistics"""

    def __init__(self, stats='numpy'):
        self.stats = stats

    def begin(self, ct, out_shape):
        img = PO.resize(ct.astype(float), out_shape).astype(np.float32)
        img, mean, std16 = PO.normalize(img, self.stats)
        return dict(img=img, labels=np.zeros(img.shape, np.uint8), kept=[], out_shape=out_shape)

    def add_roi(self, state, raters):
        res = [PO.resize(r.astype(float), state['out_shape']).astype(np.float32) for r in raters]
        v = PO.vote(res)
        kept = bool(v.sum() > 0)
        if kept:
            state['labels'][v >= 0.5] = 1 + sum(state['kept'])
        state['kept'].append(kept)

    def finish(self, state):
        lab = state['labels']
        slice_nz = (lab != 0).reshape(lab.shape[0], -1).any(axis=1)
        present = np.zeros(256, bool)
        present[np.unique(lab)] = True
        return state['img'], lab, np.array(state['kept'], bool), slice_nz, present
