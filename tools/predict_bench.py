#!/usr/bin/env python
"""Wall time of sharded test-set prediction: Predictor.predict_test_set on get_test_generator(cf, logger, rank, world_size), one process
per rank, at each world size of --worlds (default: 1 and the number of visible GPUs).  Rank r runs on cuda:(r % GPUs), over NCCL when every
rank has its own GPU, else over gloo.  Prints one JSON line per measurement, the first naming the cards and their power limits.

The test set is --patients synthetic lidc_exp patients of --shape (y, x, z) voxels, written as preprocessing.py writes them ({pid}_img.npy
float32 (z, y, x), {pid}_rois.npy uint8, meta_info pickles, info_df.pickle), with --epochs seeded Retina U-Net checkpoints (3D, 128×128×64
patches, batch 8, the mirrored passes of cf.test_aug).  The untrained nets keep every detection (model_min_confidence 0), so weighted box
clustering sees the configured maximum of boxes per patch.

Per world size, every rank first predicts one patient (warm-up), then the whole test set between two barriers: `rank_s` is a host clock
around a rank's synchronised predict_test_set call (rank 0's includes the gather and the file write), `total_s` rank 0's clock from the
first barrier to the second; `patch_forwards` counts patches x mirrors x checkpoints, `forwards_per_s` is that over total_s.
`same_file_as_world_1` compares rank 0's raw_pred_boxes file with the first world size's.

    python tools/predict_bench.py [--worlds 1,8] [--patients 16] [--shape 320 320 192] [--epochs 2] [--out-dir DIR]"""
import argparse
import hashlib
import json
import os
import pickle
import shutil
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PATCH = (128, 128, 64)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else [torch.cuda.get_device_name(0)]


def emit(**kw):
    print(json.dumps(kw), flush=True)


class _Log:
    def info(self, *a, **k):
        pass

    warning = info


def make_cf(root, epochs):
    from medicaldetectiontoolkit_b200.configs import make_cf as mk
    cf = mk('retina_unet', 3, PATCH, exp='lidc_exp', batch_size=8)
    for k, v in dict(test_aug=True, return_masks_in_test=False, wcs_iou=1e-5, merge_3D_iou=0.1, fold=0, folds=[0], test_n_epochs=epochs,
                     model_min_confidence=0.0, hold_out_test_set=True).items():
        setattr(cf, k, v)
    cf.pp_data_path = cf.pp_test_data_path = os.path.join(root, 'pp')
    cf.exp_dir = root
    return cf


def write_test_set(root, n, shape, epochs):
    """synthetic patients in preprocessing.py's files and seeded checkpoints; returns the patches per patient"""
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import preprocessing, retina_unet
    pp = os.path.join(root, 'pp')
    os.makedirs(pp)
    Y, X, Z = shape
    rs = np.random.RandomState(0)
    zz, yy, xx = np.ogrid[:Z, :Y, :X]
    for i in range(n):
        pid = '%04d' % i
        seg = np.zeros((Z, Y, X), np.uint8)
        for k in range(3):
            c = [rs.randint(8, s - 8) for s in (Z, Y, X)]
            r = rs.randint(3, 8)
            seg[((zz - c[0]) * 2) ** 2 + (yy - c[1]) ** 2 + (xx - c[2]) ** 2 <= r * r] = k + 1
        np.save(os.path.join(pp, '%s_img.npy' % pid), rs.randn(Z, Y, X).astype(np.float32))
        np.save(os.path.join(pp, '%s_rois.npy' % pid), seg)
        fg = [int(z) for z in np.nonzero(seg.reshape(Z, -1).any(1))[0]]
        with open(os.path.join(pp, 'meta_info_%s.pickle' % pid), 'wb') as f:
            pickle.dump([pid, [int(rs.randint(1, 6)) for _ in range(3)], (0.7, 0.7, 1.25), fg], f)
    preprocessing.aggregate_meta_info(pp)
    cf = make_cf(root, epochs)
    ckpt = os.path.join(root, 'checkpoints')
    for ep in range(epochs):
        torch.manual_seed(ep)
        os.makedirs(os.path.join(ckpt, '{}_best_checkpoint'.format(ep)))
        torch.save(retina_unet.net(cf, None).state_dict(), os.path.join(ckpt, '{}_best_checkpoint'.format(ep), 'params.pth'))
    np.save(os.path.join(ckpt, 'epoch_ranking.npy'), np.arange(epochs))
    return len(D.get_patch_crop_coords(np.broadcast_to(np.uint8(0), [max(s, p) for s, p in zip(shape, PATCH)]), PATCH))


def _rank(rank, world, port, root, epochs, backend, q):
    try:
        import torch.distributed as dist
        from medicaldetectiontoolkit_b200 import data_loader as D
        from medicaldetectiontoolkit_b200 import predictor, retina_unet
        dev = torch.device('cuda', rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group(backend, rank=rank, world_size=world)
        cf = make_cf(root, epochs)
        net = retina_unet.net(cf, None).to(dev)
        for tag in ('warmup', 'timed'):
            cf.fold_dir = os.path.join(root, 'w%d-%s-r%d' % (world, tag, rank))
            shutil.copytree(os.path.join(root, 'checkpoints'), cf.fold_dir)
            cf.max_test_patients = world if tag == 'warmup' else 'all'
            gen = D.get_test_generator(cf, _Log(), rank, world)
            pred = predictor.Predictor(cf, net, _Log(), 'test')
            dist.barrier()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pred.predict_test_set(gen)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            dist.barrier()
            t2 = time.perf_counter()
        digest = None
        if rank == 0:
            with open(os.path.join(cf.fold_dir, 'raw_pred_boxes_hold_out_list.pickle'), 'rb') as f:
                digest = hashlib.sha256(f.read()).hexdigest()
        dist.destroy_process_group()
        q.put((rank, {'device': str(dev), 'patients': gen['n_test'], 'rank_s': t1 - t0, 'total_s': t2 - t0, 'sha256': digest}))
    except BaseException:
        import traceback
        q.put((rank, traceback.format_exc()))


def run_world(world, root, epochs):
    backend = 'nccl' if world <= torch.cuda.device_count() else 'gloo'
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_rank, args=(r, world, port, root, epochs, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=3600) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(world):
        if not isinstance(got[r], dict):
            raise RuntimeError('world %d rank %d failed:\n%s' % (world, r, got[r]))
    return backend, [got[r] for r in range(world)]


def main():
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--worlds", default=None, help="comma-separated world sizes (default: 1 and the number of visible GPUs)")
    p.add_argument("--patients", type=int, default=16)
    p.add_argument("--shape", type=int, nargs=3, default=[320, 320, 192], metavar=('Y', 'X', 'Z'))
    p.add_argument("--epochs", type=int, default=2, help="ensembled checkpoints")
    p.add_argument("--out-dir", default=None, help="where the test set is written (default: a temporary directory, removed after)")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("predict_bench needs a CUDA device")
    n_gpu = torch.cuda.device_count()
    worlds = [int(w) for w in a.worlds.split(',')] if a.worlds else sorted({1, n_gpu})
    emit(cards=card(), visible_gpus=n_gpu, torch=torch.__version__)
    tmp = tempfile.mkdtemp(dir=a.out_dir)
    try:
        patches = write_test_set(tmp, a.patients, tuple(a.shape), a.epochs)
        forwards = a.patients * patches * 4 * a.epochs
        first = None
        for world in worlds:
            backend, ranks = run_world(world, tmp, a.epochs)
            total = ranks[0]['total_s']
            first = first or ranks[0]['sha256']
            emit(kind='predict_test_set', world=world, backend=backend, patients=a.patients, shape_yxz=a.shape, patches_per_patient=patches,
                 epochs=a.epochs, mirrors=4, patch_forwards=forwards, total_s=round(total, 3), forwards_per_s=round(forwards / total, 1),
                 ranks=[{'device': r['device'], 'patients': r['patients'], 'rank_s': round(r['rank_s'], 3)} for r in ranks],
                 same_file_as_world_1=ranks[0]['sha256'] == first)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
