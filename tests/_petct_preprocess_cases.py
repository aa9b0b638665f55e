"""Synthetic raw PET-CT directories and z-crop volumes for the PET-CT preprocessing tests, generated from fixed geometry, and a numpy
stand-in for petct_preprocessing.CudaOps.

A raw file keeps the name the reference reads (lsa_ct.nii.gz, lsa_pet.nii.gz, lsa.seg.nrrd) but holds an .npy array; its geometry sits in
the sidecar geometry.json of the patient's directory: (spacing, origin, direction) of the images in ITK's (x, y, z) order, and the pynrrd
header of the seg ('space directions' with null for the list axis of a 4-D stack, 'space origin', 'Segment{k}_Name')."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
import petct_preprocess_oracle as PO  # noqa: E402

SIDECAR = 'geometry.json'
FLIP_Y = (1, 0, 0, 0, -1, 0, 0, 0, 1)


def _ellipse(shape_yx, centre, radii):
    y, x = np.ogrid[:shape_yx[0], :shape_yx[1]]
    return ((y - centre[0]) / float(radii[0])) ** 2 + ((x - centre[1]) / float(radii[1])) ** 2 <= 1.0


def _ellipsoid(shape, centre, radii):
    g = np.ogrid[tuple(slice(0, s) for s in shape)]
    return sum(((a - c) / float(r)) ** 2 for a, c, r in zip(g, centre, radii)) <= 1.0


def ct_volume(shape, lungs, lung_z, body_radii):
    """int16 (z, y, x): air (-1000) around an elliptic body (40) with two lungs (-850) in slices lung_z, a bone block past the clip (900)
    and a patch below it (-1500)"""
    Z, Y, X = shape
    plane = np.where(_ellipse((Y, X), (Y / 2.0, X / 2.0), body_radii), 40, -1000).astype(np.int16)
    lung = np.zeros((Y, X), bool)
    for c, r in lungs:
        lung |= _ellipse((Y, X), c, r)
    v = np.broadcast_to(plane, shape).copy()
    v[lung_z[0]:lung_z[1] + 1][:, lung] = -850
    v[:, Y // 2 - 3:Y // 2 + 3, X // 2 - 2:X // 2 + 2] = 900
    v[:, :3, :3] = -1500
    return v


def pet_volume(shape, hot):
    """float32 (z, y, x): 0.25 background, 1.5 in a central box, 8.0 in the box `hot` (z, y, x slices)"""
    Z, Y, X = shape
    p = np.full(shape, 0.25, np.float32)
    p[:, Y // 4:3 * Y // 4, X // 4:3 * X // 4] = 1.5
    p[hot] = 8.0
    return p


# pid directory, CT ((z, y, x), spacing, origin, direction, lungs [((y, x), (ry, rx))], lung slices, body radii), PET ((z, y, x), spacing,
# origin, hot box), seg (4-D?, Fortran order?, (x, y, z) size, space directions diagonal, space origin, [(name, centre (x, y, z), radii)])
PATIENTS = [
    # CT below the spacing threshold (resampled); a 4-D Fortran-order stack with a background category between two foreground segments;
    # the body reaches the last slice, so z_max is past the end
    ('TNM_study_a/pat_01',
     ((100, 140, 140), (0.7, 0.7, 2.0), (-49.0, -49.0, -100.0), None, [((70, 36), (40, 28)), ((70, 104), (40, 28))], (30, 99), (62, 66)),
     ((50, 25, 25), (4.0, 4.0, 4.0), (-49.0, -49.0, -100.0), np.s_[30:38, 10:14, 6:10]),
     (True, True, (140, 140, 100), (0.7, 0.7, 2.0), (-49.0, -49.0, -100.0),
      [('T_primary', (40, 60, 70), (6, 8, 5)), ('N_inflammation', (100, 70, 50), (8, 8, 6)), ('N_1', (70, 30, 80), (5, 5, 4))])),
    # CT above the threshold (kept) with a flipped y axis; a 3-D seg with negative x / y space directions; the body starts at slice 3, so
    # the crop's z_min is negative and wraps to the last slices
    ('TNM_study_a/pat_02',
     ((60, 100, 100), (1.0, 1.0, 3.0), (-50.0, 49.0, -90.0), FLIP_Y, [((50, 25), (28, 20)), ((50, 75), (28, 20))], (3, 52), (45, 48)),
     ((45, 25, 25), (4.0, 4.0, 4.0), (-50.0, -50.0, -90.0), np.s_[40:44, 8:12, 8:12]),
     (False, False, (50, 50, 60), (-2.0, -2.0, 3.0), (50.0, 50.0, -90.0), [('T_primary', (20, 30, 57), (4, 5, 3))])),
    # a one-voxel lesion on a fine seg grid that linear resampling cannot keep (class_target == []), beside a background-category segment
    ('TNM_study_b/pat_03',
     ((80, 110, 110), (0.9, 0.9, 2.5), (-49.5, -49.5, -100.0), None, [((55, 30), (31, 22)), ((55, 80), (31, 22))], (20, 70), (50, 52)),
     ((55, 25, 25), (4.0, 4.0, 4.0), (-49.5, -49.5, -100.0), np.s_[25:30, 12:16, 12:16]),
     (True, False, (40, 40, 20), (0.45, 0.45, 1.25), (-9.0, -9.0, 10.0),
      [('T_primary', (20, 20, 10), (0.5, 0.5, 0.5)), ('M1b_brain', (20, 20, 10), (12, 12, 6))])),
]

# directories collect_paths must skip: no 'TNM' in the path, no PET file
DECOYS = [('other/pat_09', ['lsa_pet.nii.gz']), ('TNM_study_b/notes', ['readme.txt'])]


def _seg_array(size, segments, four_d, fortran):
    masks = [_ellipsoid(size, c, r).astype(np.uint8) for _, c, r in segments]
    if len(masks) == 1 and not four_d:
        arr = masks[0]
    else:
        arr = np.stack(masks)
    return np.asfortranarray(arr) if fortran else arr


def make_raw_dir(root):
    """writes root/raw/... and returns the raw data directory"""
    raw = os.path.join(root, 'raw')
    for rel, ct_spec, pet_spec, seg_spec in PATIENTS:
        d = os.path.join(raw, rel)
        os.makedirs(d)
        shape, sp, org, direction, lungs, lung_z, body = ct_spec
        direction = direction or (1, 0, 0, 0, 1, 0, 0, 0, 1)
        geom = {}

        def put(name, arr):
            with open(os.path.join(d, name), 'wb') as f:
                np.save(f, arr)
        put('lsa_ct.nii.gz', ct_volume(shape, lungs, lung_z, body))
        geom['lsa_ct.nii.gz'] = [list(sp), list(org), list(direction)]
        pshape, psp, porg, hot = pet_spec
        put('lsa_pet.nii.gz', pet_volume(pshape, hot))
        geom['lsa_pet.nii.gz'] = [list(psp), list(porg), [1, 0, 0, 0, 1, 0, 0, 0, 1]]
        four_d, fortran, size, diag, sorg, segments = seg_spec
        put('lsa.seg.nrrd', _seg_array(size, segments, four_d, fortran))
        dirs = np.diag(diag).tolist()
        header = {'type': 'unsigned char', 'dimension': 4 if four_d else 3,
                  'space directions': ([None] if four_d else []) + dirs, 'space origin': list(sorg)}
        for k, (name, _, _) in enumerate(segments):
            header['Segment%d_Name' % k] = name
            header['Segment%d_Color' % k] = '0.5 0.5 0.5'
        geom['lsa.seg.nrrd'] = header
        with open(os.path.join(d, SIDECAR), 'w') as f:
            json.dump(geom, f)
    for rel, files in DECOYS:
        d = os.path.join(raw, rel)
        os.makedirs(d)
        for name in files:
            open(os.path.join(d, name), 'w').close()
    return raw


def read_image(path):
    """read_image for the synthetic directories: (array (z, y, x), spacing, origin, direction)"""
    with open(os.path.join(os.path.dirname(path), SIDECAR)) as f:
        sp, org, direction = json.load(f)[os.path.basename(path)]
    return np.load(path), tuple(sp), tuple(org), tuple(float(v) for v in direction)


def read_seg(path):
    """read_seg for the synthetic directories: (array, header) with pynrrd's keys and array types"""
    with open(os.path.join(os.path.dirname(path), SIDECAR)) as f:
        header = json.load(f)[os.path.basename(path)]
    header['space directions'] = np.array([[np.nan] * 3 if r is None else r for r in header['space directions']], dtype=np.float64)
    header['space origin'] = np.array(header['space origin'], dtype=np.float64)
    return np.load(path), header


# ------------------------------------------------------------------------------------------------------------------- z-crop volumes
def _squares(shape, per_slice):
    """int16 (z, y, x) of 0 with -1000 squares: per_slice [((z0, z1), (y0, x0, h, w))] inclusive z ranges"""
    v = np.zeros(shape, np.int16)
    for (z0, z1), (y0, x0, h, w) in per_slice:
        v[z0:z1 + 1, y0:y0 + h, x0:x0 + w] = -1000
    return v


def zcrop_cases():
    """name -> (volume, kwargs of get_z_crops)"""
    S = (24, 24)
    c = {}
    c['settled'] = (_squares((60,) + S, [((10, 50), (3, 3, 6, 6)), ((10, 50), (14, 14, 6, 6))]), dict(min_pix=20, n_comps=2, rad_crit=200))
    # dist >= 151 first, then settled with min_pix + 500
    c['too_long'] = (_squares((200, 64, 64), [((10, 60), (5, 5, 25, 25)), ((10, 60), (34, 34, 25, 25)), ((61, 180), (10, 10, 6, 6)),
                                              ((61, 180), (40, 40, 6, 6))]), dict(min_pix=20, n_comps=2, rad_crit=2000))
    # dist <= 43 first, then settled with one component
    c['too_short'] = (_squares((60, 64, 64), [((20, 40), (5, 5, 20, 20)), ((10, 50), (34, 34, 20, 20))]), dict(min_pix=120, n_comps=2, rad_crit=2000))
    c['wraps'] = (_squares((60,) + S, [((2, 40), (3, 3, 6, 6)), ((2, 40), (14, 14, 6, 6))]), dict(min_pix=20, n_comps=2, rad_crit=200))
    c['past_end'] = (_squares((45,) + S, [((8, 44), (3, 3, 6, 6)), ((8, 44), (14, 14, 6, 6))]), dict(min_pix=20, n_comps=2, rad_crit=200))
    # slices 10..50: a square whose corner meets a border pixel diagonally (cleared by the 8-connected clear_border) and one plain square;
    # slices 20..60: two plain squares
    diag = _squares((70,) + S, [((10, 50), (1, 1, 6, 6)), ((10, 60), (14, 14, 6, 6)), ((20, 60), (14, 3, 6, 6))])
    diag[10:51, 0, 0] = -1000
    c['diagonal_border'] = (diag, dict(min_pix=20, n_comps=2, rad_crit=200))
    # slices 5..15: a square of exactly min_pix pixels; slices 20..60: two larger squares
    c['exact_min_pix'] = (_squares((70,) + S, [((5, 15), (3, 3, 5, 5)), ((5, 60), (14, 14, 6, 6)), ((20, 60), (3, 14, 6, 6))]),
                          dict(min_pix=25, n_comps=2, rad_crit=200))
    # slices 5..15: a centroid exactly at rad_crit (squared distance 100); slices 20..60: at 81
    c['exact_rad_crit'] = (_squares((70, 64, 64), [((5, 15), (30, 40, 5, 5)), ((20, 60), (30, 39, 5, 5)), ((5, 60), (30, 28, 5, 5))]),
                           dict(min_pix=20, n_comps=2, rad_crit=100))
    c['empty'] = (_squares((40,) + S, [((5, 30), (3, 3, 4, 4))]), dict(min_pix=20, n_comps=2, rad_crit=200))
    c['never_settles'] = (_squares((20,) + S, [((0, 19), (3, 3, 6, 6)), ((0, 19), (14, 14, 6, 6))]), dict(min_pix=20, n_comps=2, rad_crit=200))
    return c


# ------------------------------------------------------------------------------------------------------------------- numpy stand-in
class NumpyOps(object):
    """numpy stand-in for petct_preprocessing.CudaOps on petct_preprocess_oracle; stats='numpy' normalises as the reference does,
    stats='device' with the device's fp64 statistics"""

    def __init__(self, stats='numpy'):
        self.stats = stats

    def upload(self, arr):
        return np.ascontiguousarray(arr)

    def to_host(self, a):
        return np.asarray(a)

    def resample(self, src, in_grid, out_grid, out_dtype):
        return PO.resample(src, in_grid.as_dict(), out_grid.as_dict(), out_dtype)

    def seg_merge(self, readdata, selected):
        seg = np.zeros(readdata.shape[1:], np.uint8)
        for k, on in enumerate(selected):
            if on:
                seg[readdata[k] == 1] = 1
        return np.ascontiguousarray(seg.transpose(2, 1, 0))

    def body_components(self, ct):
        first, stats = PO.body_components(ct)
        return None, first, stats

    def zcrop_flags(self, comps, shape, min_pix, n_comps, rad_crit):
        return PO.zcrop_flags(comps[1], comps[2], shape[1], shape[2], min_pix, n_comps, rad_crit)

    def normalize(self, ct, pet):
        return (PO.normalize if self.stats == 'numpy' else PO.normalize_device)(ct, pet)

    def label_summary(self, seg):
        present = np.zeros(256, bool)
        present[np.unique(seg)] = True
        return (seg != 0).reshape(seg.shape[0], -1).any(axis=1), present
