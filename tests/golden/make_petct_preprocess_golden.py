"""Records tests/golden/petct_preprocess.pkl.gz from the reference's unmodified experiments/pet_ct_tnm_classification/preprocessing.py
(pp_patient and get_z_crops) over the synthetic cases of tests/_petct_preprocess_cases.py.

    python tests/golden/make_petct_preprocess_golden.py <reference root>

The reference module is loaded from its file with stubs installed first: SimpleITK over the cases' .npy files and geometry sidecars, its
resampling as oracle/petct_preprocess_oracle.resample (ITK's arithmetic is pinned through that restatement only), nrrd as the cases'
reader, skimage.segmentation.clear_border as the oracle's restatement, and a `configs` module.  The reference only processes the pids of
its `selection`, so every patient is passed as pid 106 and its files are collected after each call; info_df.pickle is created empty before
each call, as the reference expects it to exist.  get_z_crops is wrapped to record the crop of the outermost call.  The z-crop cases call
get_z_crops directly and record its return value or the name of the exception it raises."""
import gzip
import importlib.util
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _petct_preprocess_cases as PC  # noqa: E402
import petct_preprocess_oracle as PO  # noqa: E402  (on sys.path through _petct_preprocess_cases)

OUT = os.path.join(HERE, 'petct_preprocess.pkl.gz')
PID = 106


class _Image(object):
    """the part of sitk.Image the reference uses: a (z, y, x) array with ITK geometry"""

    def __init__(self, arr, spacing=(1.0, 1.0, 1.0), origin=(0.0, 0.0, 0.0), direction=(1, 0, 0, 0, 1, 0, 0, 0, 1)):
        self.arr = arr
        self.spacing, self.origin, self.direction = tuple(spacing), tuple(origin), tuple(float(d) for d in direction)

    def GetSpacing(self):
        return self.spacing

    def GetOrigin(self):
        return self.origin

    def GetDirection(self):
        return self.direction

    def GetSize(self):
        return tuple(self.arr.shape[::-1])

    def GetPixelIDValue(self):
        return self.arr.dtype

    def SetSpacing(self, s):
        self.spacing = tuple(float(v) for v in s)

    def SetOrigin(self, o):
        self.origin = tuple(float(v) for v in o)

    def SetDirection(self, d):
        self.direction = tuple(float(v) for v in d)

    def grid(self):
        return PO.grid(self.GetSize(), self.origin, self.spacing, self.direction)


def _resample(img, ref):
    return _Image(PO.resample(img.arr, img.grid(), ref.grid(), img.arr.dtype), ref.spacing, ref.origin, ref.direction)


class _ResampleImageFilter(object):
    def SetReferenceImage(self, ref):
        self.ref = ref

    def Execute(self, img):
        return _resample(img, self.ref)


def _install_stubs(pp):
    sitk = types.ModuleType('SimpleITK')
    sitk.ReadImage = lambda path: (lambda a, sp, org, d: _Image(a, sp, org, d))(*PC.read_image(path))
    sitk.GetArrayFromImage = lambda img: img.arr
    sitk.GetImageFromArray = lambda arr: _Image(np.ascontiguousarray(arr))
    sitk.Image = lambda size, pixel_id: _Image(np.zeros(tuple(size)[::-1], pixel_id))
    sitk.Resample = _resample
    sitk.ResampleImageFilter = _ResampleImageFilter
    nrrd = types.ModuleType('nrrd')
    nrrd.read = PC.read_seg
    skimage = types.ModuleType('skimage')
    transform = types.ModuleType('skimage.transform')
    transform.resize = None                      # imported by the reference, not called
    segmentation = types.ModuleType('skimage.segmentation')
    segmentation.clear_border = PO.clear_border
    skimage.transform, skimage.segmentation = transform, segmentation
    configs = types.ModuleType('configs')

    class _Cf(object):
        def __init__(self):
            self.pp_dir = pp
    configs.configs = _Cf
    sys.modules.update({'SimpleITK': sitk, 'nrrd': nrrd, 'skimage': skimage, 'skimage.transform': transform, 'skimage.segmentation': segmentation,
                        'configs': configs})


def _load_reference(ref_root):
    path = os.path.join(ref_root, 'experiments', 'pet_ct_tnm_classification', 'preprocessing.py')
    spec = importlib.util.spec_from_file_location('petct_preprocessing_ref', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _outcome(fn):
    try:
        return tuple(int(v) for v in fn())
    except (ValueError, RecursionError) as e:
        return type(e).__name__


def record(ref_root):
    golden = {'patients': {}, 'zcrop': {}}
    with tempfile.TemporaryDirectory() as tmp:
        raw = PC.make_raw_dir(tmp)
        pp = os.path.join(tmp, 'pp')
        os.makedirs(pp)
        _install_stubs(pp)
        mod = _load_reference(ref_root)
        inner = mod.get_z_crops
        crops = []

        def recording(*args, **kwargs):
            depth = len(crops)
            crops.append(None)
            out = inner(*args, **kwargs)
            if depth == 0:
                crops[0] = out
            return out
        mod.get_z_crops = recording
        for rel, _, _, _ in PC.PATIENTS:
            pd.DataFrame(columns=['pid', 'raw_pid', 'class_target', 'fg_slices']).to_pickle(os.path.join(pp, 'info_df.pickle'))
            del crops[:]
            mod.pp_patient((PID, os.path.join(raw, rel)))
            row = pd.read_pickle(os.path.join(pp, 'info_df.pickle')).iloc[-1].to_dict()
            golden['patients'][rel] = dict(img=np.load(os.path.join(pp, '%d_img.npy' % PID)), rois=np.load(os.path.join(pp, '%d_rois.npy' % PID)),
                                           row=row, zcrop=tuple(int(v) for v in crops[0]))
        mod.get_z_crops = inner
        for name, (vol, kw) in PC.zcrop_cases().items():
            golden['zcrop'][name] = _outcome(lambda: inner(vol, 0, **kw))
    with gzip.open(OUT, 'wb', compresslevel=9) as f:
        pickle.dump(golden, f, protocol=4)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    if len(sys.argv) != 2:
        sys.exit('usage: make_petct_preprocess_golden.py <reference root>')
    record(sys.argv[1])
