"""Goldens of the data loader (tests/golden/loader.json.gz) from the reference's own code: the unmodified BatchGenerator and
PatientBatchIterator of experiments/{lidc_exp,toy_exp,pet_ct_tnm_classification}/data_loader.py and the functions of
utils/dataloader_utils.py, on the synthetic preprocessed directories of tests/_loader_cases.py.

Run where the reference tree is present: python tests/golden/make_loader_golden.py <reference root>.  Re-running reproduces the file byte for
byte.  batchgenerators is not needed: SlimDataLoaderBase is a minimal stand-in (it stores the data and the batch size), and
ConvertSegToBoundingBoxCoordinates is the restatement oracle/augment_oracle.seg_to_boxes (get_rois_from_seg_flag=False), whose results are
stored with np.array as batchgenerators stores them.  The reference was written for numpy < 1.24: its modules see a numpy whose np.array
makes an object array of a ragged list, as numpy did then.  Each training configuration is seeded with np.random.seed([0, 0]), the stream
of data_loader.BatchGenerator(seed=0, rank=0)."""
import gzip
import io
import json
import logging
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]

import _loader_cases as LC  # noqa: E402
import augment_oracle as AO  # noqa: E402

OUT = os.path.join(HERE, 'loader.json.gz')


def _np_shim():
    shim = types.ModuleType('numpy_pre_1_24')
    shim.__dict__.update(np.__dict__)

    def array(obj, *a, **k):
        try:
            return np.array(obj, *a, **k)
        except ValueError:
            if a or k:
                raise
            out = np.empty(len(obj), dtype=object)
            for i, v in enumerate(obj):
                out[i] = v
            return out
    shim.array = array
    return shim


class SlimDataLoaderBase(object):
    def __init__(self, data, batch_size, number_of_threads_in_multithreaded=None):
        self._data = data
        self.batch_size = batch_size


class ConvertSegToBoundingBoxCoordinates(object):
    def __init__(self, dim, get_rois_from_seg_flag=False, class_specific_seg_flag=False):
        assert not get_rois_from_seg_flag
        self.dim, self.flag = dim, class_specific_seg_flag

    def __call__(self, **d):
        r = AO.seg_to_boxes(d['seg'], d['class_target'], self.dim, self.flag, with_masks=False)
        shim = _np_shim()
        d.update({'bb_target': shim.array(r['bb_target']), 'roi_labels': shim.array(r['roi_labels']), 'seg': r['seg']})
        return d


def _install_stubs(ref):
    sys.path.insert(0, ref)
    mods = {}
    for name in ('batchgenerators', 'batchgenerators.dataloading', 'batchgenerators.dataloading.data_loader',
                 'batchgenerators.dataloading.multi_threaded_augmenter', 'batchgenerators.transforms',
                 'batchgenerators.transforms.spatial_transforms', 'batchgenerators.transforms.abstract_transforms',
                 'batchgenerators.transforms.crop_and_pad_transforms', 'batchgenerators.transforms.utility_transforms', 'SimpleITK', 'preprocessing'):
        mods[name] = sys.modules[name] = types.ModuleType(name)
    mods['batchgenerators.dataloading.data_loader'].SlimDataLoaderBase = SlimDataLoaderBase
    mods['batchgenerators.dataloading'].SingleThreadedAugmenter = None
    mods['batchgenerators.dataloading.multi_threaded_augmenter'].MultiThreadedAugmenter = None
    for k in ('MirrorTransform', 'SpatialTransform'):
        setattr(mods['batchgenerators.transforms.spatial_transforms'], k, None)
    mods['batchgenerators.transforms.abstract_transforms'].Compose = None
    mods['batchgenerators.transforms.crop_and_pad_transforms'].CenterCropTransform = None
    mods['batchgenerators.transforms.utility_transforms'].ConvertSegToBoundingBoxCoordinates = ConvertSegToBoundingBoxCoordinates


def _ref_module(ref, exp):
    import importlib.util
    spec = importlib.util.spec_from_file_location('ref_loader_' + exp, os.path.join(ref, 'experiments', exp, 'data_loader.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    m.np = _np_shim()
    m.dutils.np = m.np
    return m


EXP = {'lidc': 'lidc_exp', 'pet': 'pet_ct_tnm_classification', 'toy': 'toy_exp'}


def _utils_goldens(dutils):
    out = {'fold_generator': [], 'class_balanced': [], 'patch_crop_coords': [], 'pad_nd_image': []}
    for seed, k, n in [(0, 5, 23), (3, 5, 21), (1, 4, 9), (7, 3, 3), (0, 5, 100), (2, 6, 13)]:
        out['fold_generator'].append({'args': [seed, k, n], 'folds': LC.plain(dutils.fold_generator(seed, k, n).get_fold_names())})
    rs = np.random.RandomState(5)
    for seed in range(6):
        targets = [[int(c) for c in rs.randint(0, 2, rs.randint(0, 4))] for _ in range(12)]
        np.random.seed([seed, 0])
        ixs = dutils.get_class_balanced_patients(targets, 8, 2, slack_factor=0.2)
        out['class_balanced'].append({'seed': seed, 'targets': targets, 'ixs': LC.plain(ixs)})
    for shape, ps in [((300, 280, 250), (128, 128, 64)), ((128, 128, 64), (128, 128, 64)), ((512, 512), (288, 288)), ((70, 90, 5), (32, 32, 1)),
                      ((100, 61, 40), (64, 32, 40))]:
        out['patch_crop_coords'].append({'shape': list(shape), 'patch': list(ps),
                                         'coords': LC.plain(dutils.get_patch_crop_coords(np.zeros(shape, np.uint8), ps))})
    img = np.arange(2 * 5 * 7 * 3, dtype=np.float32).reshape(2, 5, 7, 3)
    for kw in [dict(new_shape=(8, 8, 4)), dict(new_shape=(4, 9), mode='constant'), dict(new_shape=(6, 6, 6), mode='edge', return_slicer=True),
               dict(new_shape=None, shape_must_be_divisible_by=[4, 4, 4]), dict(new_shape=(5, 7, 3), shape_must_be_divisible_by=3)]:
        r = dutils.pad_nd_image(img, **kw)
        if isinstance(r, tuple):
            r = [r[0].tolist(), [[s.start, s.stop] for s in r[1]]]
        else:
            r = r.tolist()
        out['pad_nd_image'].append({'kwargs': {k: (list(v) if isinstance(v, tuple) else v) for k, v in kw.items()}, 'result': r})
    return out


def main(ref):
    _install_stubs(ref)
    mods = {k: _ref_module(ref, e) for k, e in EXP.items()}
    golden = {'utils': _utils_goldens(mods['lidc'].dutils), 'train': {}, 'patients': {}}
    log = logging.getLogger('golden')
    with tempfile.TemporaryDirectory() as tmp:
        dirs = {}
        for kind in EXP:
            dirs[kind] = os.path.join(tmp, kind)
            LC.write_dir(kind, dirs[kind])
        for name, spec in LC.CASES.items():
            kind = spec[0]
            cf = LC.case_cf(spec)
            data = LC.dataset(kind, dirs[kind])
            gen = mods[kind].BatchGenerator(data, cf.batch_size, cf)
            np.random.seed([0, 0])
            golden['train'][name] = [LC.digest(gen.generate_train_batch()) for _ in range(LC.N_BATCHES)]
        for name, spec in LC.PATIENT_CASES.items():
            kind = spec[0]
            cf = LC.case_cf(spec)
            data = LC.dataset(kind, dirs[kind])
            it = mods[kind].PatientBatchIterator(data, cf)
            golden['patients'][name] = [LC.digest(it.generate_train_batch()) for _ in range(len(data))]
        raising = os.path.join(tmp, 'raising')
        LC.write_raising_dir(raising)
        cf = LC.case_cf(LC.CASES['lidc_3d'])
        cf.head_classes = 2
        gen = mods['lidc'].BatchGenerator(LC.dataset('lidc', raising), 1, cf)
        np.random.seed([0, 0])
        for i in range(LC.N_BATCHES):
            try:
                gen.generate_train_batch()
            except ValueError as e:
                golden['raising'] = {'batch': i, 'error': str(e)}
                break
    buf = io.BytesIO()
    with gzip.GzipFile(fileobj=buf, mode='wb', mtime=0, filename='') as f:
        f.write(json.dumps(LC.plain(golden), sort_keys=True, default=lambda v: v.item()).encode())
    with open(OUT, 'wb') as f:
        f.write(buf.getvalue())
    print('wrote', OUT, len(buf.getvalue()), 'bytes; raising:', golden.get('raising'))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
