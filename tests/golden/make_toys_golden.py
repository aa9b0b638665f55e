"""Records tests/golden/toys.json.gz from the reference's unmodified experiments/toy_exp/generate_toys.py over the cases of
tests/_toys_cases.py.

    python tests/golden/make_toys_golden.py <reference root>

The reference module is imported with a stub `configs` module first on sys.path.  Each image is made by its multi_processing_create_image
after np.random.seed(key); aggregate_meta_info runs with the module's os.listdir replaced by a sorted one (the reference file itself is not
modified).  The golden keeps, per image, the sha256 of the .npy file, the meta pickle (its path relative to the experiments' root) and the
seg sum, and per split the info_df rows: hashes, not images, because fp64 noise does not compress.  Rerunning the script rewrites the file
byte for byte."""
import gzip
import hashlib
import importlib
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _toys_cases as TC  # noqa: E402

OUT = os.path.join(HERE, 'toys.json.gz')


def _load_reference(ref_root, stub_dir):
    with open(os.path.join(stub_dir, 'configs.py'), 'w') as f:
        f.write('class configs(object):\n    root_dir = None\n')
    sys.path[:0] = [stub_dir, os.path.join(ref_root, 'experiments', 'toy_exp')]
    mod = importlib.import_module('generate_toys')
    sorted_os = types.SimpleNamespace(**{k: getattr(os, k) for k in ('path', 'makedirs')})
    sorted_os.listdir = lambda d: sorted(os.listdir(d))
    mod.os = sorted_os
    return mod


def _sha256(path):
    with open(path, 'rb') as f:
        return hashlib.sha256(f.read()).hexdigest()


def record(ref_root):
    golden = {}
    with tempfile.TemporaryDirectory() as tmp:
        mod = _load_reference(ref_root, os.path.join(tmp))
        root = os.path.join(tmp, 'root')
        for name, mode, diameters, seed, n in TC.CASES:
            margin = np.max(diameters) // 2
            case = {'mode': mode, 'class_diameters': list(diameters), 'seed': seed, 'n': n}
            for s, split in enumerate(TC.SPLITS):
                out_dir = os.path.join(root, name, split)
                os.makedirs(out_dir)
                images = []
                for six in range(n):
                    np.random.seed([seed, s, six])
                    mod.multi_processing_create_image([out_dir, six, margin, diameters, mode])
                    path = os.path.join(out_dir, '%d.npy' % six)
                    with open(os.path.join(out_dir, 'meta_info_%d.pickle' % six), 'rb') as f:
                        meta = pickle.load(f)
                    images.append({'sha256': _sha256(path), 'meta': [os.path.relpath(meta[0], root), meta[1], meta[2]],
                                   'meta_types': [type(v).__name__ for v in meta], 'seg_sum': float(np.load(path)[1].sum())})
                mod.aggregate_meta_info(out_dir)
                df = pd.read_pickle(os.path.join(out_dir, 'info_df.pickle'))
                rows = [[os.path.relpath(p, root), int(c), pid] for p, c, pid in zip(df['path'], df['class_id'], df['pid'])]
                case[split] = {'images': images, 'info_df': rows, 'columns': list(df.columns)}
            golden[name] = case
    data = json.dumps(golden, sort_keys=True, indent=1).encode()
    with open(OUT, 'wb') as f:
        f.write(gzip.compress(data, compresslevel=9, mtime=0))
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    if len(sys.argv) != 2:
        sys.exit('usage: make_toys_golden.py <reference root>')
    record(sys.argv[1])
