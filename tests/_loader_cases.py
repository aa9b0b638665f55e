"""Synthetic preprocessed dataset directories in the reference loaders' format, the loader configurations the goldens of
tests/golden/make_loader_golden.py cover, a numpy stand-in for data_loader's device ops, and the batch digests both sides record."""
import hashlib
import os

import numpy as np

from medicaldetectiontoolkit_b200.configs import make_cf

N_BATCHES = 50


def _lesions(rs, seg, n, label_of, border=False, size=(2, 6)):
    Z, Y, X = seg.shape
    for k in range(n):
        ext = [int(rs.randint(size[0], size[1])) for _ in range(3)]
        lo = [int(rs.randint(0, max(1, s - e))) for s, e in zip((Z, Y, X), ext)]
        if border and k == 0:
            lo[1] = 0
        seg[lo[0]:lo[0] + ext[0], lo[1]:lo[1] + ext[1], lo[2]:lo[2] + ext[2]] = label_of(k)


def write_lidc_dir(path, seed, kind='lidc'):
    """lidc_exp ({pid}_img.npy float32 (z, y, x), {pid}_rois.npy uint8 instance ids) or pet_ct ({pid}_img.npy float16 (2, z, y, x), binary
    {pid}_rois.npy) with info_df.pickle (pid, class_target, fg_slices).  Patients: regular ones, one smaller than the pre-crop on z, one
    without foreground, one with a lesion at the y border and odd y / x extents (the fallback window), one with 255 labels."""
    import pandas as pd
    rs = np.random.RandomState(seed)
    os.makedirs(path, exist_ok=True)
    shapes = {'p0': (30, 48, 50), 'p1': (16, 60, 44), 'p2': (28, 44, 44), 'p3': (26, 43, 45), 'p4': (30, 52, 46), 'p5': (24, 42, 42)}
    rows = []
    for pid, (Z, Y, X) in shapes.items():
        seg = np.zeros((Z, Y, X), np.uint8)
        if pid == 'p4':
            ids = np.arange(1, 256, dtype=np.uint8)
            flat = seg[:Z - 2].reshape(-1)          # two empty slices: the 2D slice draw divides by the count of slices without foreground
            flat[rs.choice(flat.size, 255, replace=False)] = ids
            n = 255
        elif pid != 'p2':
            n = int(rs.randint(1, 4))
            _lesions(rs, seg, n, lambda k: k + 1, border=pid in ('p3', 'p5'))
        else:
            n = 0
        if kind == 'pet':
            seg = (seg > 0).astype(np.uint8)
            img = rs.rand(2, Z, Y, X).astype(np.float16)
            ct = int(rs.randint(0, 2))
        else:
            img = rs.randn(Z, Y, X).astype(np.float32)
            # p5 is all benign: the reference's class balancing redraws forever when no patient has more benign than malignant ROIs
            ct = [int(rs.randint(1, 3 if pid == 'p5' else 6)) for _ in range(n)]
        np.save(os.path.join(path, '%s_img.npy' % pid), img)
        np.save(os.path.join(path, '%s_rois.npy' % pid), seg)
        rows.append({'pid': pid, 'class_target': ct, 'fg_slices': [int(z) for z in np.nonzero(seg.reshape(Z, -1).any(1))[0]]})
    pd.DataFrame(rows).to_pickle(os.path.join(path, 'info_df.pickle'))


def write_toy_dir(path, seed, n=6, size=64):
    """toy_exp: {pid}.npy float64 [2, size, size] (image, seg) and info_df.pickle (pid, class_id)"""
    import pandas as pd
    rs = np.random.RandomState(seed)
    os.makedirs(path, exist_ok=True)
    rows = []
    for i in range(n):
        a = np.zeros((2, size, size))
        a[0] = rs.rand(size, size)
        lo = rs.randint(0, size - 12, 2)
        a[1, lo[0]:lo[0] + 10, lo[1]:lo[1] + 10] = 1
        np.save(os.path.join(path, 'toy%d.npy' % i), a)
        rows.append({'pid': 'toy%d' % i, 'class_id': int(rs.randint(0, 2))})
    pd.DataFrame(rows).to_pickle(os.path.join(path, 'info_df.pickle'))


def write_raising_dir(path):
    """one lidc patient (sampled with head_classes = 2: np.random.choice, no class balancing) whose fallback window draws randint(20, 20): y extent 41 with pre-crop 40, a lesion at y = 0"""
    import pandas as pd
    os.makedirs(path, exist_ok=True)
    seg = np.zeros((30, 41, 50), np.uint8)
    seg[10:14, 0:4, 20:24] = 1
    np.save(os.path.join(path, 'q0_img.npy'), np.zeros(seg.shape, np.float32))
    np.save(os.path.join(path, 'q0_rois.npy'), seg)
    pd.DataFrame([{'pid': 'q0', 'class_target': [3], 'fg_slices': list(range(10, 14))}]).to_pickle(os.path.join(path, 'info_df.pickle'))


# name -> (dataset kind, make_cf arguments, overrides)
CASES = {
    'lidc_3d': ('lidc', ('retina_unet', 3, (32, 32, 16), 'lidc_exp'), {'pre_crop_size': [40, 40, 24], 'batch_size': 4}),
    'lidc_2d': ('lidc', ('mrcnn', 2, (32, 32), 'lidc_exp'), {'pre_crop_size': [40, 40], 'batch_size': 6}),
    'lidc_2d_ctx': ('lidc', ('mrcnn', 2, (32, 32), 'lidc_exp'), {'pre_crop_size': [40, 40], 'batch_size': 6, 'n_3D_context': 2}),
    'pet_3d': ('pet', ('retina_unet', 3, (32, 32, 16), 'pet_ct_tnm_classification'), {'pre_crop_size': [40, 40, 24], 'batch_size': 4}),
    'pet_2d_ctx': ('pet', ('retina_unet', 2, (32, 32), 'pet_ct_tnm_classification'), {'pre_crop_size': [40, 40], 'batch_size': 6,
                                                                                      'n_3D_context': 1}),
    'toy_2d': ('toy', ('mrcnn', 2, (64, 64), 'toy_exp'), {'pre_crop_size': [64, 64], 'batch_size': 4}),
}
# PatientBatchIterator cases.  A patient smaller than the patch has no golden: the reference pads its seg with the data's 4-entry new_shape
# and raises IndexError (pad_nd_image indexes the seg's 3-entry shape with it).
PATIENT_CASES = {
    'lidc_3d_patients': ('lidc', ('retina_unet', 3, (32, 32, 16), 'lidc_exp'), {}),
    'lidc_2d_patients': ('lidc', ('mrcnn', 2, (32, 32), 'lidc_exp'), {'n_3D_context': 1}),
    'lidc_2d_nomerge': ('lidc', ('mrcnn', 2, (32, 32), 'lidc_exp'), {'merge_2D_to_3D_preds': False}),
    'toy_patients': ('toy', ('mrcnn', 2, (64, 64), 'toy_exp'), {}),
}


def case_cf(spec):
    kind, args, over = spec
    cf = make_cf(args[0], args[1], args[2], exp=args[3])
    for k, v in over.items():
        setattr(cf, k, v)
    return cf


def write_dir(kind, path, seed=0):
    if kind == 'toy':
        write_toy_dir(path, seed)
    else:
        write_lidc_dir(path, seed, kind)


def dataset(kind, path):
    """the OrderedDict load_dataset builds for the case's directory"""
    import logging
    from medicaldetectiontoolkit_b200.data_loader import load_dataset
    cf = make_cf(exp={'lidc': 'lidc_exp', 'pet': 'pet_ct_tnm_classification', 'toy': 'toy_exp'}[kind], dim=2)
    cf.pp_data_path = path
    cf.select_prototype_subset = None
    return load_dataset(cf, logging.getLogger('loader'))


# ------------------------------------------------------------------------------------------------------------------- digests
def plain(x):
    """nested Python lists / ints / floats / strings of a batch entry (object arrays element by element)"""
    if isinstance(x, np.ndarray) and x.dtype == object:
        return [plain(v) for v in x]
    if isinstance(x, np.ndarray):
        return x.tolist()
    if isinstance(x, (list, tuple)):
        return [plain(v) for v in x]
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, np.generic):
        return x.item()
    return x


def _arr(x):
    if hasattr(x, 'detach'):
        x = x.detach().cpu().numpy()
    x = np.ascontiguousarray(x)
    return {'shape': list(x.shape), 'dtype': str(x.dtype), 'sha256': hashlib.sha256(x.tobytes()).hexdigest()}


def digest(batch):
    out = {}
    for k in sorted(batch):
        if k in ('data', 'seg'):
            out[k] = _arr(batch[k])
        elif k == 'roi_masks':
            continue
        elif k == 'pid':
            out[k] = plain(batch[k]) if isinstance(batch[k], (list, tuple)) else str(batch[k])
        else:
            out[k] = plain(batch[k])
    return out


# ------------------------------------------------------------------------------------------------------------------- numpy ops
class NumpyOps(object):
    """numpy stand-in for data_loader.CudaOps: the foreground index from np.argwhere order, the gather by fancy indexing"""

    def fg_index(self, seg):
        t = np.transpose(seg, (1, 2, 0)).reshape(-1)
        counts = np.bincount(t, minlength=256).astype(np.int64)
        fg = np.flatnonzero(t)
        return counts, fg[np.argsort(t[fg], kind='stable')]

    def upload(self, arr):
        return np.ascontiguousarray(arr)

    def gather(self, src, elems, tabs, out_dtype, key='src'):
        flat = np.concatenate([np.ascontiguousarray(w).reshape(-1) for w in src]) if isinstance(src, list) else src.reshape(-1)
        tab_c, tab_z, tab_y, tab_x = [np.asarray(t, np.int64) for t in tabs]
        n, C = tab_c.shape
        I, J, K = tab_y.shape[1], tab_x.shape[1], tab_z.shape[2]
        out = np.zeros((n, C, I, J, K), dtype=out_dtype)
        for b in range(n):
            e = elems[b]
            ext = (int(e['c']), int(e['z']), int(e['y']), int(e['x']))
            vol = flat[int(e['offset']):int(e['offset']) + int(np.prod(ext))].reshape(ext)
            idx = [tab_c[b][:, None, None, None], tab_z[b][:, None, None, :], tab_y[b][None, :, None, None], tab_x[b][None, None, :, None]]
            ok = np.ones((C, I, J, K), dtype=bool)
            for t, s in zip(idx, ext):
                ok &= (t >= 0) & (t < s)
            v = vol[tuple(np.clip(t, 0, s - 1) for t, s in zip(idx, ext))]
            out[b] = np.where(ok, v.astype(out_dtype), np.zeros((), out_dtype))
        return out

    def seg_to_boxes(self, seg, lut):
        B = seg.shape[0]
        stats = np.zeros((B, 255, 7), np.int32)
        stats[:, :, 1:4] = 0x7fffffff
        stats[:, :, 4:7] = -1
        for b in range(B):
            s = seg[b, 0]
            for k in np.unique(s):
                if k == 0:
                    continue
                ix = np.argwhere(s == k)
                st = stats[b, k - 1]
                st[0] = len(ix)
                st[1:1 + ix.shape[1]] = ix.min(0)
                st[4:4 + ix.shape[1]] = ix.max(0)
            if s.ndim == 2:
                stats[b, :, 3] = np.where(stats[b, :, 0] > 0, 0, stats[b, :, 3])
                stats[b, :, 6] = np.where(stats[b, :, 0] > 0, 0, stats[b, :, 6])
        out = np.take_along_axis(lut[:, None, :], seg.reshape(B, 1, -1).astype(np.int64), axis=2).reshape(seg.shape)
        return stats, out

    def to_host(self, x):
        return x
