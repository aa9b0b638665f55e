"""data_loader's host side against the goldens of the reference's own loaders (tests/golden/make_loader_golden.py): the dataloader_utils
restatements, and BatchGenerator / PatientBatchIterator with a numpy stand-in for the device ops, digest for digest."""
import gzip
import json
import os

import numpy as np
import pytest

import _loader_cases as LC
from medicaldetectiontoolkit_b200 import data_loader as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'loader.json.gz')


@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN) as f:
        return json.loads(f.read())


@pytest.fixture(scope='module')
def dirs(tmp_path_factory):
    root = tmp_path_factory.mktemp('loader')
    out = {}
    for kind in ('lidc', 'pet', 'toy'):
        out[kind] = str(root / kind)
        LC.write_dir(kind, out[kind])
    out['raising'] = str(root / 'raising')
    LC.write_raising_dir(out['raising'])
    return out


def test_fold_generator(golden):
    for g in golden['utils']['fold_generator']:
        assert LC.plain(D.fold_generator(*g['args']).get_fold_names()) == g['folds'], g['args']


def test_class_balanced_patients(golden):
    for g in golden['utils']['class_balanced']:
        rs = np.random.RandomState([g['seed'], 0])
        assert LC.plain(D.get_class_balanced_patients(g['targets'], 8, 2, slack_factor=0.2, rs=rs)) == g['ixs']


def test_patch_crop_coords(golden):
    for g in golden['utils']['patch_crop_coords']:
        assert LC.plain(D.get_patch_crop_coords(np.zeros(g['shape'], np.uint8), g['patch'])) == g['coords']


def test_pad_nd_image(golden):
    img = np.arange(2 * 5 * 7 * 3, dtype=np.float32).reshape(2, 5, 7, 3)
    for g in golden['utils']['pad_nd_image']:
        kw = {k: (tuple(v) if isinstance(v, list) and k == 'new_shape' else v) for k, v in g['kwargs'].items()}
        r = D.pad_nd_image(img, **kw)
        r = [r[0].tolist(), [[s.start, s.stop] for s in r[1]]] if isinstance(r, tuple) else r.tolist()
        assert r == g['result'], kw


@pytest.mark.parametrize('name', sorted(LC.CASES))
def test_batch_generator_digests(golden, dirs, name):
    spec = LC.CASES[name]
    cf = LC.case_cf(spec)
    gen = D.BatchGenerator(LC.dataset(spec[0], dirs[spec[0]]), cf.batch_size, cf, seed=0, rank=0, ops=LC.NumpyOps())
    for i, want in enumerate(golden['train'][name]):
        assert LC.digest(gen.generate_train_batch()) == want, (name, i)


@pytest.mark.parametrize('name', sorted(LC.PATIENT_CASES))
def test_patient_batch_iterator_digests(golden, dirs, name):
    spec = LC.PATIENT_CASES[name]
    cf = LC.case_cf(spec)
    it = D.PatientBatchIterator(LC.dataset(spec[0], dirs[spec[0]]), cf, ops=LC.NumpyOps())
    for i, want in enumerate(golden['patients'][name]):
        assert LC.digest(it.generate_train_batch()) == want, (name, i)


def test_fallback_window_raises(golden, dirs):
    """an axis of 41 with pre-crop 40 and a lesion at its edge: the fallback draws randint(20, 20), which raises as in the reference"""
    cf = LC.case_cf(LC.CASES['lidc_3d'])
    cf.head_classes = 2
    gen = D.BatchGenerator(LC.dataset('lidc', dirs['raising']), 1, cf, seed=0, rank=0, ops=LC.NumpyOps())
    for _ in range(golden['raising']['batch']):
        gen.generate_train_batch()
    with pytest.raises(ValueError, match=golden['raising']['error']):
        gen.generate_train_batch()


def test_server_env_is_not_supported(dirs):
    cf = LC.case_cf(LC.CASES['lidc_3d'])
    cf.server_env = True
    with pytest.raises(NotImplementedError):
        D.load_dataset(cf, None)


def test_make_cf_loader_attributes():
    """the loader attributes of experiments/{lidc_exp,toy_exp,pet_ct_tnm_classification}/configs.py (outside server_env)"""
    from medicaldetectiontoolkit_b200.configs import make_cf
    lidc3, lidc2 = make_cf('retina_unet', 3, exp='lidc_exp'), make_cf('mrcnn', 2, exp='lidc_exp')
    assert (lidc3.pre_crop_size, lidc2.pre_crop_size) == ([156, 156, 96], [300, 300])
    assert (lidc3.val_mode, lidc3.num_val_batches, lidc3.select_prototype_subset, lidc3.hold_out_test_set) == ('val_sampling', 50, 100, False)
    toy = make_cf('mrcnn', 2, (320, 320), exp='toy_exp')
    assert (toy.pre_crop_size, toy.val_mode, toy.max_val_patients, toy.hold_out_test_set, toy.merge_2D_to_3D_preds, toy.n_train_val_data) == \
        ([320, 320], 'val_patient', None, True, False, 1500)
    pet = make_cf('retina_unet', 3, exp='pet_ct_tnm_classification')
    assert (pet.pre_crop_size, pet.num_val_batches, pet.hold_out_test_set) == ([280, 280, 48], 10, True)
    for cf in (lidc3, toy, pet):
        assert (cf.seed, cf.batch_sample_slack, cf.n_3D_context, cf.max_test_patients, cf.input_df_name) == (0, 0.2, None, 'all', 'info_df.pickle')
