"""Test-set prediction sharded over a process group on the GPU: a toy experiment generated on the device (generate_toys), two seeded
Retina U-Net checkpoints and one Mask R-CNN checkpoint (return_masks_in_test) saved from cuda:0, and predict_test_set through
get_test_generator(cf, logger, rank, world_size) at world 1 and world 2 (gloo).  Rank 0's raw_pred_boxes file must be byte-identical to the
world-1 run's, its consolidated results equal, and the Evaluator's scores on them the same.

World 2 runs with both ranks on cuda:0, so one GPU suffices; with two or more GPUs visible it also runs on cuda:0 / cuda:1, where rank 1
loads checkpoints saved from cuda:0 onto its own device (map_location).  With one GPU that case is skipped and stays unverified."""
import os
import pickle
import shutil
import socket
import sys
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_TEST = 5
MODELS = {'retina_unet': (11, 12), 'mrcnn': (21,)}        # model -> the seeds of its checkpoints, best first


class _Log:
    def info(self, *a, **k):
        pass

    warning = info


def _cf(model, root):
    from medicaldetectiontoolkit_b200.configs import make_cf
    cf = make_cf(model, 2, (320, 320), exp='toy_exp', batch_size=4)
    for k, v in dict(test_aug=True, return_masks_in_test=model == 'mrcnn', wcs_iou=1e-5, fold=0, folds=[0], test_n_epochs=len(MODELS[model]),
                     model_min_confidence=0.0).items():         # an untrained net scores below the default 0.1: keep its detections
        setattr(cf, k, v)
    cf.pp_data_path = os.path.join(root, 'donuts_shape', 'train')
    cf.pp_test_data_path = os.path.join(root, 'donuts_shape', 'test')
    cf.exp_dir = root
    return cf


def _net(model, cf):
    from medicaldetectiontoolkit_b200 import mrcnn, retina_unet
    return (retina_unet if model == 'retina_unet' else mrcnn).net(cf, None)


@pytest.fixture(scope='module')
def root(tmp_path_factory):
    from medicaldetectiontoolkit_b200 import generate_toys as G
    root = str(tmp_path_factory.mktemp('predict_dist_gpu'))
    G.generate_experiment(root, 'donuts_shape', 4, N_TEST, 'donuts_shape', seed=9)
    for model, seeds in MODELS.items():
        ckpt = os.path.join(root, 'checkpoints', model)
        for ep, seed in enumerate(seeds):
            torch.manual_seed(seed)
            net = _net(model, _cf(model, root)).to('cuda:0')
            os.makedirs(os.path.join(ckpt, '{}_best_checkpoint'.format(ep)))
            torch.save(net.state_dict(), os.path.join(ckpt, '{}_best_checkpoint'.format(ep), 'params.pth'))
        np.save(os.path.join(ckpt, 'epoch_ranking.npy'), np.arange(len(seeds)))
    torch.cuda.synchronize()
    return root


def _worker(rank, world, devices, port, root, tag, q):
    try:
        sys.path.insert(0, ROOT)
        import torch.distributed as dist
        from medicaldetectiontoolkit_b200 import data_loader as D
        from medicaldetectiontoolkit_b200 import evaluator, predictor
        dev = torch.device(devices[rank])
        torch.cuda.set_device(dev)
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group('gloo', rank=rank, world_size=world)
        res = {}
        for model in MODELS:
            cf = _cf(model, root)
            cf.fold_dir = os.path.join(root, 'runs', '{}-{}-r{}'.format(model, tag, rank))
            shutil.copytree(os.path.join(root, 'checkpoints', model), cf.fold_dir)
            net = _net(model, cf).to(dev)
            gen = D.get_test_generator(cf, _Log(), rank, world)
            out = predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(gen)
            torch.cuda.synchronize()
            r = {'pids': list(gen['test'].dataset_pids), 'files': sorted(os.listdir(cf.fold_dir)), 'results': None, 'stats': None, 'raw': None,
                 'device': str(next(net.parameters()).device)}
            if out is not None:
                r['results'] = pickle.dumps(out)
                with open(os.path.join(cf.fold_dir, 'raw_pred_boxes_hold_out_list.pickle'), 'rb') as f:
                    r['raw'] = f.read()
                ev = evaluator.Evaluator(cf, _Log(), mode='test')
                ev.evaluate_predictions(out)
                r['stats'] = ev.return_metrics()[0]
            if world == 1:
                # today's unsharded generator: the same file
                cf.fold_dir += '-plain'
                shutil.copytree(os.path.join(root, 'checkpoints', model), cf.fold_dir)
                predictor.Predictor(cf, net, _Log(), 'test').predict_test_set(D.get_test_generator(cf, _Log()), return_results=False)
                with open(os.path.join(cf.fold_dir, 'raw_pred_boxes_hold_out_list.pickle'), 'rb') as f:
                    r['raw_plain'] = f.read()
            res[model] = r
        dist.destroy_process_group()
        q.put((rank, res))
    except BaseException:
        q.put((rank, traceback.format_exc()))


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _spawn(devices, root, tag):
    world = len(devices)
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, devices, port, root, tag, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=900) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(world):
        assert isinstance(got[r], dict), '{} rank {} failed:\n{}'.format(tag, r, got[r])
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [got[r] for r in range(world)]


@pytest.fixture(scope='module')
def world1(root):
    return _spawn(['cuda:0'], root, 'w1')


def test_world1_equals_the_unsharded_generator(world1):
    for model in MODELS:
        assert world1[0][model]['raw'] == world1[0][model]['raw_plain'], model


def _same_as_world1(world1, ranks, root):
    all_pids = sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(root, 'donuts_shape', 'test')) if f.endswith('.npy'))
    for model in MODELS:
        one, r0 = world1[0][model], ranks[0][model]
        assert sorted(pickle.loads(one['raw'])[i][1] for i in range(N_TEST)) == all_pids
        assert r0['raw'] == one['raw'], model
        assert r0['results'] == one['results'], model
        np.testing.assert_equal(r0['stats'], one['stats'])
        assert any(bx['box_type'] == 'det' for p in pickle.loads(one['raw']) for b in p[0] for bx in b), model
        assert sorted(ranks[0][model]['pids'] + ranks[1][model]['pids']) == sorted(one['pids'])
        assert ranks[1][model]['results'] is None and ranks[1][model]['raw'] is None
        assert 'raw_pred_boxes_hold_out_list.pickle' not in ranks[1][model]['files']


def test_world2_on_one_gpu_equals_world1(root, world1):
    ranks = _spawn(['cuda:0', 'cuda:0'], root, 'w2-one-gpu')
    _same_as_world1(world1, ranks, root)
    print('world 2 ran with both ranks on cuda:0')


def test_world2_on_two_gpus_equals_world1(root, world1):
    if torch.cuda.device_count() < 2:
        pytest.skip('one GPU visible: the cross-device run (checkpoints saved from cuda:0 loaded on cuda:1) is unverified')
    ranks = _spawn(['cuda:0', 'cuda:1'], root, 'w2-two-gpus')
    assert all(ranks[1][m]['device'] == 'cuda:1' for m in MODELS)
    _same_as_world1(world1, ranks, root)
    print('world 2 ran on cuda:0 and cuda:1')
