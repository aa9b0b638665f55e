"""LIDC preprocessing on the GPU: the reference's experiments/lidc_exp/preprocessing.py (resample_array, pp_patient, aggregate_meta_info and
its __main__) with the resampling, CT normalisation and rater vote in csrc/preprocess.cu.

It turns the raw LIDC directory of the LIDC-IDRI conversion tool ({pid}/{pid}_ct_scan.nrrd, one {pid}_..._{nodule id}_{roi id}.nii.gz per
rater annotation, characteristics.csv beside the data directory) into the directory data_loader.load_dataset reads: {pid}_img.npy (float32,
(z, y, x)), {pid}_rois.npy (uint8), meta_info_{pid}.pickle, info_df.pickle and its copy info_df_bk.pickle, and suppressed_rois.txt.

    python -m medicaldetectiontoolkit_b200.preprocessing --raw-data-dir ROOT/data_nrrd --pp-dir OUT [--root-dir ROOT]

What it computes, per patient:
  - CT: skimage.transform.resize (scikit-image 0.16.2, order 1, mode 'edge', anti-aliasing on) to target_spacing, clip to [-1200, 600],
    then (x - mean) / std with std rounded to fp16.  The device takes the mean and population std of the clipped volume in fp64 (fixed
    reduction trees, the same bits on every run) and rounds them to fp32 (the std then to fp16).  The reference takes numpy's float32
    np.mean / np.std, whose pairwise float32 sums can differ from these in the last bits of the mean.
  - ROIs: every rater mask resampled like the CT; per ROI the raters' float32 mean over max(4, raters) (zero volumes pad to four), kept
    where >= 0.5.  A ROI with no kept voxel is suppressed: its file names go to suppressed_rois.txt (space-separated, no newline, as the
    reference writes them) and it gets no label; otherwise it takes the next label, later ROIs overwriting earlier ones.  Its malignancy
    label is the mean of the raters' Malignancy in characteristics.csv, padded with zeros to four raters.

Deterministic choices where the reference's order depends on the hash seed or the file system:
  - ROI ids are processed in sorted (string) order;
  - directory listings are sorted: patients, the rater files of a ROI and the meta_info files that make info_df.
Everything else follows the reference, including the selection of a ROI's rater files by the substring '{roi id}.nii' (id 1 also takes
the files of id 11).  A patient without ROI files gets an all-zero label map and fg_slices == [].  Sources other than uint8, int16 and
float32 are rejected before any launch.

Reading .nrrd and .nii.gz files needs SimpleITK, imported only when the default reader is used; any read_image(path) -> (array (z, y, x),
spacing (x, y, z)) can replace it."""
import argparse
import ctypes
import os
import pickle
import shutil

import numpy as np
import numpy.testing as npt
import torch

from . import _lib as L

_DTYPES = {np.dtype(np.uint8): 0, np.dtype(np.int16): 4, np.dtype(np.float32): 2}   # MDT_DTYPE_U8, MDT_DTYPE_I16, MDT_DTYPE_F32
_TORCH_DTYPES = {torch.uint8: 0, torch.int16: 4, torch.float32: 2}
META_COLUMNS = ['pid', 'class_target', 'spacing', 'fg_slices']


def sitk_read_image(path):
    """(array (z, y, x), spacing (x, y, z)) of a file SimpleITK reads"""
    try:
        import SimpleITK as sitk
    except ImportError as e:
        raise ImportError("reading LIDC .nrrd / .nii.gz files needs SimpleITK (pip install SimpleITK); or pass read_image=") from e
    img = sitk.ReadImage(path)
    return sitk.GetArrayFromImage(img), img.GetSpacing()


def target_shape(shape, src_spacing, target_spacing):
    """the resampled (z, y, x) extents: source spacing (x, y, z) rounded to 3 decimals, int(extent * spacing / target) per axis"""
    src_zyx = np.round(src_spacing, 3)[::-1]
    tgt_zyx = tuple(target_spacing)[::-1]
    out = [int(n * s / t) for n, s, t in zip(shape, src_zyx, tgt_zyx)]
    if min(out) <= 0:
        raise AssertionError("AssertionError:", shape, src_spacing, target_spacing)
    return out


def _check_source(arr):
    if arr.ndim != 3:
        raise ValueError("preprocessing resamples (z, y, x) volumes; got shape %s" % (arr.shape,))
    if arr.dtype not in _DTYPES:
        raise ValueError("preprocessing resamples uint8, int16 or float32 volumes; got %s (convert it first)" % arr.dtype)


class CudaOps(object):
    """the device side of one patient: resample + normalise the CT, resample and vote each ROI's raters, summarise the label map"""

    def __init__(self, device=None):
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())

    def upload(self, arr):
        _check_source(arr)
        return torch.from_numpy(np.ascontiguousarray(arr)).to(self.device)

    def resample(self, src, out_shape, out=None):
        """src: device tensor (z, y, x) of uint8 / int16 / float32 -> float32 (out_shape)"""
        dt = _TORCH_DTYPES.get(src.dtype)
        if dt is None or src.dim() != 3 or not src.is_contiguous():
            raise ValueError("resample takes a contiguous (z, y, x) uint8, int16 or float32 tensor; got %s %s" % (src.dtype, tuple(src.shape)))
        L.require_cuda(src)
        ins = (_int3(src.shape), _int3(out_shape))
        lib = L.load()
        with torch.cuda.device(self.device):
            ws_bytes = lib.mdt_pp_resample_workspace_bytes(*ins)
            ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=self.device)
            if out is None:
                out = torch.empty(tuple(int(s) for s in out_shape), dtype=torch.float32, device=self.device)
            L.check(lib.mdt_pp_resample(dt, L.ptr(src), ins[0], ins[1], L.ptr(out), L.ptr(ws), ws_bytes, L.stream_ptr()))
        return out

    def normalize(self, img):
        """clip and normalise img (float32, device) in place; returns the device stats [mean, std] (fp64, before rounding)"""
        lib = L.load()
        with torch.cuda.device(self.device):
            n = img.numel()
            ws = torch.empty(lib.mdt_pp_normalize_workspace_bytes(n), dtype=torch.uint8, device=self.device)
            stats = torch.empty(2, dtype=torch.float64, device=self.device)
            L.check(lib.mdt_pp_normalize(L.ptr(img), n, L.ptr(stats), L.ptr(ws), ws.numel(), L.stream_ptr()))
        return stats

    def begin(self, ct, out_shape):
        img = self.resample(self.upload(ct), out_shape)
        stats = self.normalize(img)
        return dict(img=img, stats=stats, labels=torch.zeros(img.shape, dtype=torch.uint8, device=self.device),
                    kept=torch.zeros(255, dtype=torch.int32, device=self.device), acc=None, rater=None, n_rois=0)

    def add_roi(self, state, raters):
        lib = L.load()
        if state['n_rois'] > 254:
            raise ValueError("a patient can have at most 255 labelled ROIs in a uint8 label map")
        img = state['img']
        if state['acc'] is None:
            state['acc'] = torch.empty_like(img)
            state['rater'] = torch.empty_like(img)
        acc, tmp = state['acc'], state['rater']
        with torch.cuda.device(self.device):
            for k, r in enumerate(raters):
                self.resample(self.upload(r), img.shape, out=tmp)
                L.check(lib.mdt_pp_vote_add(L.ptr(acc), L.ptr(tmp), img.numel(), int(k == 0), L.stream_ptr()))
            L.check(lib.mdt_pp_vote_label(L.ptr(acc), img.numel(), len(raters), state['n_rois'], L.ptr(state['labels']), L.ptr(state['kept']),
                                          L.stream_ptr()))
        state['n_rois'] += 1

    def finish(self, state):
        """host (img float32, labels uint8, kept [n_rois] bool, slice_nz [z] bool, present [256] bool); one synchronisation"""
        lab = state['labels']
        lib = L.load()
        with torch.cuda.device(self.device):
            slice_nz = torch.empty(lab.shape[0], dtype=torch.uint8, device=self.device)
            present = torch.empty(256, dtype=torch.uint8, device=self.device)
            L.check(lib.mdt_pp_label_summary(L.ptr(lab), lab.shape[0], lab[0].numel(), L.ptr(slice_nz), L.ptr(present), L.stream_ptr()))
            out = (state['img'].cpu().numpy(), lab.cpu().numpy(), state['kept'][:state['n_rois']].cpu().numpy() != 0,
                   slice_nz.cpu().numpy() != 0, present.cpu().numpy() != 0)
        return out


def _int3(shape):
    return (ctypes.c_int * 3)(*[int(s) for s in shape])


def resample_array(src_imgs, src_spacing, target_spacing, ops=None):
    """the reference's resample_array on the device: src_imgs (z, y, x) uint8 / int16 / float32, spacings (x, y, z) -> float32 array"""
    _check_source(src_imgs)
    ops = ops or CudaOps()
    shape = target_shape(src_imgs.shape, src_spacing, target_spacing)
    return ops.resample(ops.upload(src_imgs), shape).cpu().numpy()


def _roi_groups(files):
    """(roi id, its rater files) per ROI id in sorted order; files: the sorted listing of a patient's directory"""
    ids = sorted({f.split('.')[0].split('_')[-1] for f in files if '.nii.gz' in f})
    return [(rid, [f for f in files if '{}.nii'.format(rid) in f]) for rid in ids]


def pp_patient(inputs, cf, read_image=None, ops=None):
    """one patient directory (ix, path) -> cf.pp_dir/{pid}_img.npy, {pid}_rois.npy, meta_info_{pid}.pickle (+ suppressed_rois.txt)"""
    import pandas as pd
    _, path = inputs
    read_image = read_image or sitk_read_image
    ops = ops or CudaOps()
    pid = os.path.basename(path)
    ct, ct_spacing = read_image(os.path.join(path, '{}_ct_scan.nrrd'.format(pid)))
    _check_source(ct)
    shape = target_shape(ct.shape, ct_spacing, cf.target_spacing)
    state = ops.begin(ct, shape)

    chars = pd.read_csv(os.path.join(cf.root_dir, 'characteristics.csv'), sep=';')
    chars = chars[chars.PatientID == pid]
    mal_labels, names = [], []
    for _, rater_files in _roi_groups(sorted(os.listdir(path))):
        scores = [chars[chars.NoduleID == int(f.split('_')[2].lstrip('0'))].Malignancy.values[0] for f in rater_files]
        scores += [0] * (4 - len(scores))
        mal_labels.append(np.mean([s for s in scores if s > -1]))
        raters = []
        for f in rater_files:
            arr, sp = read_image(os.path.join(cf.raw_data_dir, pid, f))
            arr = arr.astype(np.uint8)
            if target_shape(arr.shape, sp, cf.target_spacing) != shape:
                raise AssertionError([f, arr.shape, ct.shape, pid, sp])
            for a in range(3):
                npt.assert_almost_equal(sp[a], ct_spacing[a])
            raters.append(arr)
        ops.add_roi(state, raters)
        names.append(rater_files)

    img, labels, kept, slice_nz, present = ops.finish(state)
    class_target = []
    for k, rater_files in enumerate(names):
        if kept[k]:
            class_target.append(mal_labels[k])
        else:
            with open(os.path.join(cf.pp_dir, 'suppressed_rois.txt'), 'a') as f:
                f.write(' '.join(rater_files))
    class_target = np.array(class_target)
    assert len(class_target) + 1 == int(present.sum()), [len(class_target), np.flatnonzero(present), pid]
    fg_slices = [np.int64(z) for z in np.flatnonzero(slice_nz)]

    np.save(os.path.join(cf.pp_dir, '{}_rois.npy'.format(pid)), labels)
    np.save(os.path.join(cf.pp_dir, '{}_img.npy'.format(pid)), img)
    with open(os.path.join(cf.pp_dir, 'meta_info_{}.pickle'.format(pid)), 'wb') as f:
        pickle.dump({'pid': pid, 'class_target': class_target, 'spacing': ct_spacing, 'fg_slices': fg_slices}, f)


def aggregate_meta_info(exp_dir):
    """info_df.pickle from the meta_info_*.pickle files of exp_dir (in sorted name order); returns the DataFrame"""
    import pandas as pd
    rows = []
    for name in sorted(os.listdir(exp_dir)):
        if 'meta_info' in name:
            with open(os.path.join(exp_dir, name), 'rb') as f:
                rows.append(pickle.load(f))
    df = pd.DataFrame(columns=META_COLUMNS)
    for row in rows:
        df.loc[len(df)] = row
    df.to_pickle(os.path.join(exp_dir, 'info_df.pickle'))
    return df


def preprocess_lidc(cf, read_image=None, ops=None):
    """every patient of cf.raw_data_dir (sorted) into cf.pp_dir on one device, then info_df.pickle and its copy info_df_bk.pickle"""
    ops = ops or CudaOps()
    paths = [os.path.join(cf.raw_data_dir, p) for p in sorted(os.listdir(cf.raw_data_dir))]
    os.makedirs(cf.pp_dir, exist_ok=True)
    for ix, path in enumerate(paths):
        pp_patient((ix, path), cf, read_image=read_image, ops=ops)
    df = aggregate_meta_info(cf.pp_dir)
    shutil.copyfile(os.path.join(cf.pp_dir, 'info_df.pickle'), os.path.join(cf.pp_dir, 'info_df_bk.pickle'))
    return df


def main(argv=None):
    from .configs import make_cf
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--raw-data-dir', required=True, help='directory of one sub-directory per patient')
    p.add_argument('--pp-dir', required=True, help='output directory (created if missing)')
    p.add_argument('--root-dir', default=None, help='directory of characteristics.csv (default: the parent of --raw-data-dir)')
    a = p.parse_args(argv)
    cf = make_cf(exp='lidc_exp')
    cf.raw_data_dir = a.raw_data_dir
    cf.pp_dir = a.pp_dir
    cf.root_dir = a.root_dir or os.path.dirname(os.path.abspath(a.raw_data_dir))
    df = preprocess_lidc(cf)
    print("aggregated meta info to df with length", len(df))


if __name__ == '__main__':
    main()
