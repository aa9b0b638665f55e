"""PET-CT preprocessing on the GPU: the reference's experiments/pet_ct_tnm_classification/preprocessing.py (get_z_crops, pp_patient,
collectPaths and its __main__) with the resampling, segment merge, body z-crop scan and normalisation in csrc/petct_preprocess.cu.

It turns a raw directory of patient directories (each with lsa_ct.nii.gz, lsa_pet.nii.gz and the segment stack lsa.seg.nrrd, below a path
containing 'TNM') into the directory data_loader.load_dataset reads for cf.experiment == 'pet_ct_tnm_classification': {pid}_img.npy
(float32, (2, z, y, x): CT, PET), {pid}_rois.npy (uint8, (z, y, x), 0 / 1) and info_df.pickle (pid, raw_pid, class_target, fg_slices).

    python -m medicaldetectiontoolkit_b200.petct_preprocessing --raw-data-dir RAW --pp-dir OUT

What it computes, per patient:
  - Seg: the segments whose name (header keys containing '_Name') is not a background category are merged into one binary map; the
    reference's `seg[...] = ix = 1` writes 1 for every segment, so the map is binary and class_target is [labels[0]] or [].  Its grid is
    |diagonal of 'space directions'|, 'space origin' * sign(spacing) and the identity direction.
  - CT: resampled onto spacing (0.976562, 0.976562, 3.27) (size int(size * spacing / new spacing), the CT's origin and direction) when its
    x spacing is below 0.95 or its z spacing below 3.  PET and seg are resampled onto the (possibly new) CT grid, each keeping its pixel
    type.  Resampling is ITK's ResampleImageFilter with the identity transform and linear interpolation, evaluated per voxel in fp64 (ITK
    itself accumulates the continuous index along a scan line, so SimpleITK's last bits are not claimed); 0 outside the input.
  - z-crop: get_z_crops.  The per-slice components (x < -600, clear_border with 8-connectivity, then 4-connected components) and their
    count, row sum and column sum are computed once per patient on the device; each recursion level is one small criterion launch, and the
    recursion itself runs in Python as the reference's does, with the same failures: no qualifying slice raises ValueError (np.min([])), a
    recursion that never settles raises RecursionError.  The crop [z_min:z_max] has Python slice semantics: a negative z_min wraps.
  - Normalisation: CT clip(-1200, 600), (1200 + x) / 1800, (x - mean) / std in fp64, rounded to float32; PET (p - mean) / std in float32.
    The device takes the means and population stds through fixed fp64 reduction trees (the same bits on every run); the reference takes
    numpy's pairwise sums (fp64 for the CT, float32 for the PET), which can differ in the last bits.  The CT must be int16 and the PET
    float32 (their NIfTI types); other types are rejected before any launch.

Deliberate differences from the reference, whose driver is tied to one machine:
  - every patient is processed (the reference keeps a debugging selection of pids 106 and 273);
  - patient directories are taken in sorted path order, and pid is the index in that order (the reference uses os.walk's order);
  - info_df.pickle is written once, in pid order, after the last patient (the reference's eight workers rewrite a pre-existing file).

Readers are pluggable: read_image(path) -> (array (z, y, x), spacing, origin, direction), by default a lazily imported SimpleITK;
read_seg(path) -> (array, header with pynrrd's keys), by default a lazily imported pynrrd."""
import argparse
import ctypes
import os

import numpy as np
import torch

from . import _lib as L

BACKGROUND_CATEGORIES = ['M1b_brain', 'N_inflammation', 'T_benign', 'T_other']
NEW_SPACING = (0.976562, 0.976562, 3.27)
IDENTITY = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)
INFO_COLUMNS = ['pid', 'raw_pid', 'class_target', 'fg_slices']
_DTYPES = {np.dtype(np.uint8): 0, np.dtype(np.int16): 4, np.dtype(np.float32): 2}   # MDT_DTYPE_U8, MDT_DTYPE_I16, MDT_DTYPE_F32
_TORCH = {np.dtype(np.uint8): torch.uint8, np.dtype(np.int16): torch.int16, np.dtype(np.float32): torch.float32}


def sitk_read_image(path):
    """(array (z, y, x), spacing, origin, direction) of a file SimpleITK reads"""
    try:
        import SimpleITK as sitk
    except ImportError as e:
        raise ImportError("reading .nii.gz files needs SimpleITK (pip install SimpleITK); or pass read_image=") from e
    img = sitk.ReadImage(path)
    return sitk.GetArrayFromImage(img), img.GetSpacing(), img.GetOrigin(), img.GetDirection()


def nrrd_read_seg(path):
    """(array, header) of a .seg.nrrd file as pynrrd reads it"""
    try:
        import nrrd
    except ImportError as e:
        raise ImportError("reading .seg.nrrd files needs pynrrd (pip install pynrrd); or pass read_seg=") from e
    return nrrd.read(path)


class Grid(object):
    """an ITK image geometry: size, origin, spacing in (x, y, z) order and the row-major 3x3 direction"""

    def __init__(self, size, origin, spacing, direction=IDENTITY):
        self.size = tuple(int(s) for s in size)
        self.origin = tuple(float(o) for o in origin)
        self.spacing = tuple(float(s) for s in spacing)
        self.direction = tuple(float(d) for d in np.asarray(direction, dtype=np.float64).reshape(9))
        if min(self.size) < 1 or not min(self.spacing) > 0:
            raise ValueError("a grid needs sizes >= 1 and spacings > 0, got %s and %s" % (self.size, self.spacing))

    @classmethod
    def of(cls, arr_shape, spacing, origin, direction):
        return cls(tuple(arr_shape)[::-1], origin, spacing, direction)

    @property
    def shape(self):
        """(z, y, x)"""
        return self.size[::-1]

    def as_dict(self):
        return {'size': self.size, 'origin': self.origin, 'spacing': self.spacing, 'direction': self.direction}

    def c_struct(self):
        return L.PetctGrid((ctypes.c_int * 3)(*self.size), (ctypes.c_double * 3)(*self.origin), (ctypes.c_double * 3)(*self.spacing),
                           (ctypes.c_double * 9)(*self.direction))


def new_ct_grid(ct_grid):
    """the reference's CT target grid when the x spacing is below 0.95 or the z spacing below 3, else None"""
    sp = ct_grid.spacing
    if not (sp[0] < 0.95 or sp[2] < 3):
        return None
    size = [int(ct_grid.size[a] * sp[a] / NEW_SPACING[a]) for a in range(3)]
    return Grid(size, ct_grid.origin, NEW_SPACING, ct_grid.direction)


def _check_dtype(arr, what):
    dt = np.dtype(str(arr.dtype).replace('torch.', ''))
    if dt not in _DTYPES:
        raise ValueError("%s must be uint8, int16 or float32, got %s (convert it first)" % (what, dt))
    return dt


class CudaOps(object):
    """the device side of pp_patient and get_z_crops on one CUDA device"""

    def __init__(self, device=None):
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())

    def upload(self, arr):
        if torch.is_tensor(arr):
            L.require_cuda(arr)
            return arr.contiguous()
        _check_dtype(arr, 'a volume')
        return torch.from_numpy(np.ascontiguousarray(arr)).to(self.device)

    def to_host(self, t):
        return t.cpu().numpy()

    def resample(self, src, in_grid, out_grid, out_dtype):
        """src (z, y, x) device tensor on in_grid -> (z, y, x) device tensor of out_dtype on out_grid"""
        sdt, odt = _check_dtype(src, 'the resampled volume'), np.dtype(out_dtype)
        if odt not in _DTYPES:
            raise ValueError("resample writes uint8, int16 or float32, got %s" % odt)
        if tuple(src.shape) != in_grid.shape:
            raise ValueError("source shape %s does not match its grid %s" % (tuple(src.shape), in_grid.shape))
        with torch.cuda.device(self.device):
            out = torch.empty(out_grid.shape, dtype=_TORCH[odt], device=self.device)
            gi, go = in_grid.c_struct(), out_grid.c_struct()
            L.check(L.load().mdt_petct_resample(_DTYPES[sdt], L.ptr(src), ctypes.byref(gi), _DTYPES[odt], L.ptr(out), ctypes.byref(go), L.stream_ptr()))
        return out

    def seg_merge(self, readdata, selected):
        """readdata (n_seg, x, y, z) host array (C or Fortran order), selected [n_seg] bool -> binary uint8 (z, y, x) device tensor"""
        dt = _check_dtype(readdata, 'the segment stack')
        n, X, Y, Z = readdata.shape
        if len(selected) != n:
            raise ValueError("one selection flag per segment: %d flags for %d segments" % (len(selected), n))
        if not (readdata.flags.c_contiguous or readdata.flags.f_contiguous):
            readdata = np.ascontiguousarray(readdata)
        base = readdata if readdata.flags.c_contiguous else readdata.T        # pynrrd's Fortran-order arrays are read in place
        strides = (ctypes.c_longlong * 4)(*[st // readdata.itemsize for st in readdata.strides])
        sel = (ctypes.c_ubyte * n)(*[int(bool(s)) for s in selected])
        with torch.cuda.device(self.device):
            src = torch.from_numpy(np.ascontiguousarray(base)).to(self.device)
            out = torch.empty((Z, Y, X), dtype=torch.uint8, device=self.device)
            L.check(L.load().mdt_petct_seg_merge(_DTYPES[dt], L.ptr(src), n, X, Y, Z, strides, sel, L.ptr(out), L.stream_ptr()))
        return out

    def body_components(self, ct):
        """ct (z, y, x) device tensor -> (label, slice_first, stats) device tensors of mdt_petct_body_components"""
        dt = _check_dtype(ct, 'the CT')
        Z, Y, X = (int(s) for s in ct.shape)
        lib = L.load()
        with torch.cuda.device(self.device):
            cap = lib.mdt_petct_body_components_capacity(Z, Y, X)
            if cap < 1:
                raise ValueError("volume %s is too large for the component labelling (fewer than 2^31 voxels)" % ((Z, Y, X),))
            ws_bytes = lib.mdt_petct_body_components_workspace_bytes(Z, Y, X)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
            label = torch.empty((Z, Y, X), dtype=torch.int32, device=self.device)
            first = torch.empty(Z + 1, dtype=torch.int32, device=self.device)
            stats = torch.empty((cap, 3), dtype=torch.int64, device=self.device)
            L.check(lib.mdt_petct_body_components(_DTYPES[dt], L.ptr(ct), Z, Y, X, L.ptr(label), L.ptr(first), L.ptr(stats), cap, L.ptr(ws), ws_bytes,
                                                  L.stream_ptr()))
        return label, first, stats

    def zcrop_flags(self, comps, shape, min_pix, n_comps, rad_crit):
        """[Z] host bool: the slices get_z_crops keeps for these parameters"""
        _, first, stats = comps
        Z, Y, X = shape
        with torch.cuda.device(self.device):
            flags = torch.empty(Z, dtype=torch.uint8, device=self.device)
            L.check(L.load().mdt_petct_zcrop_criterion(L.ptr(first), L.ptr(stats), Z, Y, X, int(min_pix), int(n_comps), float(rad_crit), L.ptr(flags),
                                                       L.stream_ptr()))
            return flags.cpu().numpy() != 0

    def normalize(self, ct, pet):
        """cropped ct (int16) and pet (float32) device tensors of one shape -> float32 (2, z, y, x) device tensor"""
        if ct.dtype != torch.int16 or pet.dtype != torch.float32:
            raise ValueError("the normalisation takes an int16 CT and a float32 PET, got %s and %s" % (ct.dtype, pet.dtype))
        if ct.shape != pet.shape:
            raise ValueError("CT and PET shapes differ: %s and %s" % (tuple(ct.shape), tuple(pet.shape)))
        n = ct.numel()
        lib = L.load()
        with torch.cuda.device(self.device):
            out = torch.empty((2,) + tuple(ct.shape), dtype=torch.float32, device=self.device)
            if n == 0:
                return out
            ws = torch.empty(lib.mdt_petct_normalize_workspace_bytes(n), dtype=torch.uint8, device=self.device)
            stats = torch.empty(4, dtype=torch.float64, device=self.device)
            L.check(lib.mdt_petct_normalize(L.ptr(ct.contiguous()), L.ptr(pet.contiguous()), n, L.ptr(out), L.ptr(stats), L.ptr(ws), ws.numel(),
                                            L.stream_ptr()))
        return out

    def label_summary(self, seg):
        """seg (z, y, x) uint8 device tensor -> host (slice_nz [z] bool, present [256] bool)"""
        Z = int(seg.shape[0])
        if Z == 0 or seg.numel() == 0:
            return np.zeros(Z, bool), np.zeros(256, bool)
        with torch.cuda.device(self.device):
            slice_nz = torch.empty(Z, dtype=torch.uint8, device=self.device)
            present = torch.empty(256, dtype=torch.uint8, device=self.device)
            L.check(L.load().mdt_pp_label_summary(L.ptr(seg.contiguous()), Z, seg[0].numel(), L.ptr(slice_nz), L.ptr(present), L.stream_ptr()))
            return slice_nz.cpu().numpy() != 0, present.cpu().numpy() != 0


def _z_crops(ops, comps, shape, min_pix, n_comps, rad_crit):
    final_slices = [int(z) for z in np.flatnonzero(ops.zcrop_flags(comps, shape, min_pix, n_comps, rad_crit))]
    z_min = np.min(final_slices) - 7
    z_max = np.max(final_slices) + 7
    dist = z_max - z_min
    if dist >= 151:
        z_min, z_max = _z_crops(ops, comps, shape, min_pix + 500, 2, rad_crit - 500)
    if dist <= 43:
        z_min, z_max = _z_crops(ops, comps, shape, min_pix - 100, 1, rad_crit + 100)
    return z_min, z_max


def get_z_crops(x, ix, min_pix=1500, n_comps=2, rad_crit=20000, ops=None):
    """the reference's get_z_crops: (z_min, z_max) of the body in the CT x (z, y, x; host array or device tensor).  ix (the patient index)
    is only reported by the reference.  ValueError when no slice qualifies, RecursionError when the recursion does not settle."""
    ops = ops or CudaOps()
    dev = ops.upload(x)
    return _z_crops(ops, ops.body_components(dev), tuple(int(s) for s in x.shape), min_pix, n_comps, rad_crit)


def _slab(z_min, z_max, Z):
    start, stop, _ = slice(int(z_min), int(z_max)).indices(Z)
    return start, max(start, stop)


def seg_grid_and_selection(readdata, header):
    """(readdata as (n_seg, x, y, z), the seg's Grid, labels, selected flags) as pp_patient derives them from a pynrrd header"""
    if readdata.ndim == 3:
        readdata = readdata[None]
        spacing = np.diagonal(np.asarray(header['space directions'], dtype=np.float64))
    else:
        spacing = np.diagonal(np.asarray(header['space directions'], dtype=np.float64)[1:, :])
    origin = np.asarray(header['space origin'], dtype=np.float64) * np.sign(spacing)
    labels = [header[k].split('=')[-1] for k in header.keys() if '_Name' in k]
    selected = [labels[k] not in BACKGROUND_CATEGORIES for k in range(readdata.shape[0])]
    return readdata, Grid(readdata.shape[1:], origin, np.abs(spacing)), labels, selected


def process_patient(ct, ct_geom, pet, pet_geom, readdata, header, ops=None, ix=0):
    """one patient's arrays -> (img float32 (2, z, y, x), rois uint8 (z, y, x), class_target, fg_slices); *_geom = (spacing, origin,
    direction) as read_image returns them"""
    ops = ops or CudaOps()
    if np.dtype(ct.dtype) != np.int16 or np.dtype(pet.dtype) != np.float32:
        raise ValueError("the CT must be int16 and the PET float32, got %s and %s" % (ct.dtype, pet.dtype))
    readdata, s_grid, labels, selected = seg_grid_and_selection(readdata, header)
    _check_dtype(readdata, 'the segment stack')
    seg = ops.seg_merge(readdata, selected)
    x_grid = Grid.of(ct.shape, *ct_geom)
    x = ops.upload(ct)
    new = new_ct_grid(x_grid)
    if new is not None:
        x = ops.resample(x, x_grid, new, ct.dtype)
        x_grid = new
    p = ops.resample(ops.upload(pet), Grid.of(pet.shape, *pet_geom), x_grid, pet.dtype)
    s = ops.resample(seg, s_grid, x_grid, np.uint8)
    zmin, zmax = _z_crops(ops, ops.body_components(x), x_grid.shape, 1500, 2, 20000)
    lo, hi = _slab(zmin, zmax, x_grid.shape[0])
    s = s[lo:hi]
    img = ops.to_host(ops.normalize(x[lo:hi], p[lo:hi]))
    slice_nz, present = ops.label_summary(s)
    class_target = [ii for k, ii in enumerate(labels) if k + 1 < 256 and present[k + 1]]
    fg_slices = [np.int64(z) for z in np.flatnonzero(slice_nz)]
    return img, ops.to_host(s), class_target, fg_slices


def pp_patient(inputs, cf, read_image=None, read_seg=None, ops=None):
    """one patient directory (ix, path) -> cf.pp_dir/{ix}_img.npy and {ix}_rois.npy; returns its info_df row"""
    ix, path = inputs
    read_image = read_image or sitk_read_image
    read_seg = read_seg or nrrd_read_seg
    ct, *ct_geom = read_image(os.path.join(path, 'lsa_ct.nii.gz'))
    pet, *pet_geom = read_image(os.path.join(path, 'lsa_pet.nii.gz'))
    readdata, header = read_seg(os.path.join(path, 'lsa.seg.nrrd'))
    img, rois, class_target, fg_slices = process_patient(ct, ct_geom, pet, pet_geom, readdata, header, ops=ops, ix=ix)
    np.save(os.path.join(cf.pp_dir, '{}_rois.npy'.format(ix)), rois)
    np.save(os.path.join(cf.pp_dir, '{}_img.npy'.format(ix)), img)
    return {'pid': ix, 'raw_pid': path.split('/')[-1], 'class_target': class_target, 'fg_slices': fg_slices}


def collect_paths(in_dir):
    """the patient directories below in_dir (a path containing 'TNM', with a file containing 'lsa_pet'), sorted"""
    paths = []
    for path, dirs, files in os.walk(in_dir):
        pet_files = [f for f in files if 'lsa_pet' in f]
        if len(files) > 0 and 'TNM' in path and len(pet_files) > 0:
            paths.append(path)
    return sorted(paths)


def preprocess_petct(cf, read_image=None, read_seg=None, ops=None):
    """every patient of cf.raw_data_dir (collect_paths order) into cf.pp_dir on one device, then info_df.pickle; returns the DataFrame"""
    import pandas as pd
    ops = ops or CudaOps()
    os.makedirs(cf.pp_dir, exist_ok=True)
    rows = [pp_patient((ix, path), cf, read_image=read_image, read_seg=read_seg, ops=ops) for ix, path in enumerate(collect_paths(cf.raw_data_dir))]
    df = pd.DataFrame(columns=INFO_COLUMNS)
    for row in rows:
        df.loc[len(df)] = row
    df.to_pickle(os.path.join(cf.pp_dir, 'info_df.pickle'))
    return df


def main(argv=None):
    from .configs import make_cf
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--raw-data-dir', required=True, help='directory searched for TNM patient directories')
    p.add_argument('--pp-dir', required=True, help='output directory (created if missing)')
    a = p.parse_args(argv)
    cf = make_cf(exp='pet_ct_tnm_classification')
    cf.raw_data_dir = a.raw_data_dir
    cf.pp_dir = a.pp_dir
    df = preprocess_petct(cf)
    print("wrote %d patients to %s" % (len(df), a.pp_dir))


if __name__ == '__main__':
    main()
