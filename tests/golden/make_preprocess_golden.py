"""Records tests/golden/preprocess.pkl.gz from the reference's unmodified experiments/lidc_exp/preprocessing.py (pp_patient and
aggregate_meta_info) over the synthetic raw directory of tests/_preprocess_cases.py.

    python tests/golden/make_preprocess_golden.py <reference root>

The reference module is loaded from its file with stubs installed first: SimpleITK over the cases' .npy files and spacing sidecars,
skimage.transform.resize as oracle/preprocess_oracle.resize (scikit-image is not a dependency here), and a `configs` module.  The module's
own `set` and `os.listdir` are replaced by versions that iterate in sorted order, so that the ROI and file orders do not depend on the
hash seed or the file system; the reference file itself is not modified."""
import builtins
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
import _preprocess_cases as PC  # noqa: E402
import preprocess_oracle as PO  # noqa: E402  (on sys.path through _preprocess_cases)

OUT = os.path.join(HERE, 'preprocess.pkl.gz')


class _Image(object):
    def __init__(self, arr, spacing):
        self.arr, self.spacing = arr, spacing

    def GetSpacing(self):
        return self.spacing


def _install_stubs(root, raw, pp):
    sitk = types.ModuleType('SimpleITK')
    sitk.ReadImage = lambda path: _Image(*PC.npy_reader(path))
    sitk.GetArrayFromImage = lambda img: img.arr
    skimage = types.ModuleType('skimage')
    transform = types.ModuleType('skimage.transform')

    def resize(image, output_shape, order=1, clip=True, mode='edge'):
        assert order == 1 and clip and mode == 'edge'
        return PO.resize(image, output_shape)
    transform.resize = resize
    skimage.transform = transform
    configs = types.ModuleType('configs')

    class _Cf(object):
        def __init__(self):
            self.root_dir, self.raw_data_dir, self.pp_dir = root, raw, pp
            self.target_spacing = PC.TARGET_SPACING
    configs.configs = _Cf
    sys.modules.update({'SimpleITK': sitk, 'skimage': skimage, 'skimage.transform': transform, 'configs': configs})


def _load_reference(ref_root):
    path = os.path.join(ref_root, 'experiments', 'lidc_exp', 'preprocessing.py')
    spec = importlib.util.spec_from_file_location('lidc_preprocessing', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sorted_os = types.SimpleNamespace(**{k: getattr(os, k) for k in ('path', 'mkdir')})
    sorted_os.listdir = lambda d: sorted(os.listdir(d))
    mod.os = sorted_os
    mod.set = lambda items: sorted(builtins.set(items))
    return mod


def record(ref_root):
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, 'root')
        raw = PC.make_raw_dir(root)
        pp = os.path.join(tmp, 'pp')
        os.makedirs(pp)
        _install_stubs(root, raw, pp)
        mod = _load_reference(ref_root)
        for ix, pid in enumerate(sorted(os.listdir(raw))):
            mod.pp_patient((ix, os.path.join(raw, pid)))
        mod.aggregate_meta_info(pp)
        golden = {'patients': {}, 'info_df': {}}
        for pid in sorted(os.listdir(raw)):
            with open(os.path.join(pp, 'meta_info_%s.pickle' % pid), 'rb') as f:
                meta = pickle.load(f)
            golden['patients'][pid] = dict(img=np.load(os.path.join(pp, '%s_img.npy' % pid)), rois=np.load(os.path.join(pp, '%s_rois.npy' % pid)),
                                           meta=meta)
        df = pd.read_pickle(os.path.join(pp, 'info_df.pickle'))
        golden['info_df'] = {c: list(df[c]) for c in df.columns}
        with open(os.path.join(pp, 'suppressed_rois.txt')) as f:
            golden['suppressed'] = f.read()
    with gzip.open(OUT, 'wb', compresslevel=9) as f:
        pickle.dump(golden, f, protocol=4)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    if len(sys.argv) != 2:
        sys.exit('usage: make_preprocess_golden.py <reference root>')
    record(sys.argv[1])
