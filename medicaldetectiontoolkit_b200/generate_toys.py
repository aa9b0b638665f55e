"""The toy experiment's data on the GPU: the reference's experiments/toy_exp/generate_toys.py (multi_processing_create_image,
generate_experiment, aggregate_meta_info and its __main__) with the images drawn by csrc/toys.cu.

It writes the directory data_loader.load_dataset reads for cf.experiment == 'toy_exp': {root_dir}/{exp_name}/{train,test}/ with {six}.npy
(float64 [2, 320, 320]: the image, then the seg as 0.0 / 1.0), meta_info_{six}.pickle ([npy path, class_id, str(six)]) and info_df.pickle
(columns path, class_id, pid).

    python -m medicaldetectiontoolkit_b200.generate_toys --root-dir ROOT [--seed S]

One deliberate difference: image six of split s (0 = train, 1 = test) draws from np.random.RandomState([seed, s, six]) (numpy's
init_by_array on the three words) instead of numpy's unseeded global state in a pool of worker processes.  An image's bytes therefore depend
only on its key, not on how images are batched or which run wrote them.  Everything after the seeding follows the reference, including a
class diameter used as a radius, discs of radius max(diameters) cut by the border (the margin is half of it), and the hole of a donut drawn
even where it lies outside a small disc.  info_df's rows follow the sorted listing of the meta_info files, not the file system's order."""
import argparse
import operator
import os
import pickle

import numpy as np
import torch

from . import _lib as L

SIDE = 320
CHUNK = 128            # images per launch: 210 MB of fp64 output on the device and in the pinned host buffer
HOLE, HOLE_CLEARS_SEG = 1, 2   # MDT_TOY_HOLE, MDT_TOY_HOLE_CLEARS_SEG
META_COLUMNS = ['path', 'class_id', 'pid']
EXPERIMENTS = [('donuts_shape', 'donuts_shape', (20, 20)), ('donuts_pattern', 'donuts_pattern', (20, 20)),
               ('circles_scale', 'circles_scale', (19, 20))]


def margin_of(class_diameters):
    """generate_experiment's foreground margin, max(class_diameters) // 2; ValueError where randint(margin, 320 - margin) would raise one,
    or for diameters that are not non-negative integers"""
    ds = [operator.index(d) for d in class_diameters]
    if len(ds) < 2 or min(ds) < 0 or max(ds) >= 2 ** 31:
        raise ValueError("class_diameters must hold at least two integers in [0, 2^31); got %r" % (tuple(class_diameters),))
    margin = max(ds) // 2
    if margin >= SIDE - margin:
        raise ValueError("low >= high: a foreground margin of %d leaves no centre in a %d-pixel image" % (margin, SIDE))
    return margin


def mode_flags(mode):
    """'donuts' in mode draws the hole of class 1; mode == 'donuts_shape' also clears the seg there"""
    return (HOLE if 'donuts' in mode else 0) | (HOLE_CLEARS_SEG if mode == 'donuts_shape' else 0)


def _keys(keys):
    k = np.asarray(keys)
    if k.ndim != 2 or k.shape[1] != 3 or k.shape[0] < 1 or k.dtype.kind not in 'iu':
        raise ValueError("keys must be a non-empty integer array [n, 3]; got %s %s" % (k.dtype, k.shape))
    if (k < 0).any() or (k > 2 ** 32 - 1).any():
        raise ValueError("key words must lie in [0, 2^32)")
    return np.ascontiguousarray(k.astype(np.uint32))


class CudaOps(object):
    """the device side: launches of mdt_toy_images and the pinned host buffer the images are copied through"""

    def __init__(self, device=None):
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())

    def images(self, keys, mode, class_diameters, margin):
        """keys uint32 [n, 3] -> device (img float64 [n, 2, 320, 320], params int32 [n, 3] = (center_x, center_y, class_id))"""
        n = keys.shape[0]
        with torch.cuda.device(self.device):
            k = torch.from_numpy(keys.view(np.int32)).to(self.device)
            img = torch.empty((n, 2, SIDE, SIDE), dtype=torch.float64, device=self.device)
            params = torch.empty((n, 3), dtype=torch.int32, device=self.device)
            L.check(L.load().mdt_toy_images(L.ptr(k), n, margin, int(class_diameters[0]), int(class_diameters[1]), mode_flags(mode),
                                            L.ptr(img), L.ptr(params), L.stream_ptr()))
        return img, params

    def staging(self, n):
        return torch.empty((n, 2, SIDE, SIDE), dtype=torch.float64, pin_memory=True)


def create_images(keys, mode, class_diameters=(20, 20), device=None):
    """the images of keys (integers [n, 3], one RandomState key per image) with generate_experiment's margin: device tensors
    (img float64 [n, 2, 320, 320], params int32 [n, 3] = (center_x, center_y, class_id))"""
    margin = margin_of(class_diameters)
    keys = _keys(keys)
    return CudaOps(device).images(keys, mode, class_diameters, margin)


def _write(out_dir, six, arr, class_id):
    out_path = os.path.join(out_dir, '{}.npy'.format(six))
    np.save(out_path, arr)
    with open(os.path.join(out_dir, 'meta_info_{}.pickle'.format(six)), 'wb') as handle:
        pickle.dump([out_path, class_id, str(six)], handle)


def generate_experiment(root_dir, exp_name, n_train_images, n_test_images, mode, class_diameters=(20, 20), seed=0, ops=None):
    """{root_dir}/{exp_name}/{train,test}: n_train_images and n_test_images images with their meta_info pickles and info_df.pickle.
    Images go in launches of CHUNK through one pinned host buffer; the next launch runs while a chunk's files are written."""
    margin = margin_of(class_diameters)
    if not 0 <= operator.index(seed) <= 2 ** 32 - 1:
        raise ValueError("seed must lie in [0, 2^32); got %d" % seed)
    dirs = [os.path.join(root_dir, exp_name, s) for s in ('train', 'test')]
    for d in dirs:
        os.makedirs(d, exist_ok=True)
    jobs = [(0, six) for six in range(n_train_images)] + [(1, six) for six in range(n_test_images)]
    if jobs:
        ops = ops or CudaOps()
        chunks = [jobs[i:i + CHUNK] for i in range(0, len(jobs), CHUNK)]
        launch = lambda chunk: ops.images(np.array([[seed, s, six] for s, six in chunk], dtype=np.uint32), mode, class_diameters, margin)
        host = ops.staging(len(chunks[0]))
        host_np = host.numpy()
        pending = launch(chunks[0])
        for k, chunk in enumerate(chunks):
            img, params = pending
            host[:len(chunk)].copy_(img)
            params = params.cpu().numpy()
            del img
            pending = launch(chunks[k + 1]) if k + 1 < len(chunks) else None
            for i, (s, six) in enumerate(chunk):
                _write(dirs[s], six, host_np[i], int(params[i, 2]))
    for d in dirs:
        aggregate_meta_info(d)


def aggregate_meta_info(exp_dir):
    """info_df.pickle from the meta_info_*.pickle files of exp_dir, in sorted name order; returns the DataFrame"""
    import pandas as pd
    rows = []
    for name in sorted(os.listdir(exp_dir)):
        if 'meta_info' in name:
            with open(os.path.join(exp_dir, name), 'rb') as handle:
                rows.append(pickle.load(handle))
    df = pd.DataFrame(columns=META_COLUMNS)
    for row in rows:
        df.loc[len(df)] = row
    df.to_pickle(os.path.join(exp_dir, 'info_df.pickle'))
    return df


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--root-dir', required=True, help='directory the experiments are written to (created if missing)')
    p.add_argument('--seed', type=int, default=0, help='the experiments draw from seeds S, S + 1 and S + 2')
    a = p.parse_args(argv)
    for k, (name, mode, diameters) in enumerate(EXPERIMENTS):
        generate_experiment(a.root_dir, name, n_train_images=1500, n_test_images=1000, mode=mode, class_diameters=diameters, seed=a.seed + k)
        print('wrote', os.path.join(a.root_dir, name))


if __name__ == '__main__':
    main()
