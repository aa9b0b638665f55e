"""Test-set prediction sharded over a gloo process group on the CPU: data_loader.get_test_generator(cf, logger, rank, world_size) and
Predictor.predict_test_set on its shard, at world sizes 1, 2 and 3.

The patients come from the synthetic preprocessed directories of tests/_loader_cases.py through the real loader with its numpy stand-in
for the device ops; the network is the deterministic stand-in of tests/test_predictor_cpu.py (its detections depend on the loaded
checkpoint), and weighted_box_clustering / nms_2to3D are bound to oracle/consolidate_oracle.py as there.  The cases cover 3D and 2D,
patched and unpatched patients, test_aug on and off, two ensembled checkpoints, merge_2D_to_3D_preds, the fold split and the hold-out
directory, and a max_test_patients cap smaller than the world."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPOCHS = (7, 3)                 # epoch_ranking.npy: two ensembled checkpoints
WORLDS = (1, 2, 3)


class _Log:
    def info(self, *a, **k):
        pass

    warning = info


# name -> (make_cf arguments, overrides, directory).  'lidc' test patients are the fold split of exp/fold_ids.pickle.
CASES = {
    'lidc_3d_patched_aug': (('retina_unet', 3, (32, 32, 16), 'lidc_exp'), dict(test_aug=True, hold_out_test_set=False), 'lidc'),
    'lidc_2d_merge_holdout': (('mrcnn', 2, (32, 32), 'lidc_exp'), dict(test_aug=False, n_3D_context=1, hold_out_test_set=True), 'lidc'),
    'toy_2d_unpatched_aug': (('retina_unet', 2, (64, 64), 'toy_exp'), dict(test_aug=True), 'toy'),
    'lidc_3d_unpatched_capped': (('retina_unet', 3, (64, 64, 32), 'lidc_exp'), dict(test_aug=False, hold_out_test_set=True, max_test_patients=2),
                                 'lidc'),
}
UNCAPPED = [c for c in CASES if 'max_test_patients' not in CASES[c][1]]
TEST_IX = [0, 1, 2, 4, 5]      # the fold's test split: 5 of the 6 lidc patients


def _case_cf(name, root):
    from medicaldetectiontoolkit_b200.configs import make_cf
    args, over, d = CASES[name]
    cf = make_cf(args[0], args[1], args[2], exp=args[3], batch_size=3)
    for k, v in dict(wcs_iou=1e-5, merge_3D_iou=0.1, test_n_epochs=len(EPOCHS), folds=[0], fold=0, return_masks_in_test=False).items():
        setattr(cf, k, v)
    for k, v in over.items():
        setattr(cf, k, v)
    cf.pp_data_path = cf.pp_test_data_path = os.path.join(root, d)
    cf.exp_dir = os.path.join(root, 'exp')
    return cf


def _write_inputs(root):
    import _loader_cases as LC
    LC.write_lidc_dir(os.path.join(root, 'lidc'), seed=3)
    LC.write_toy_dir(os.path.join(root, 'toy'), seed=4, n=5, size=64)
    os.makedirs(os.path.join(root, 'exp'))
    with open(os.path.join(root, 'exp', 'fold_ids.pickle'), 'wb') as f:
        pickle.dump([[np.array([3]), np.array([]), np.array(TEST_IX), 0]], f)
    ckpt = os.path.join(root, 'checkpoints')
    for ep in EPOCHS:
        os.makedirs(os.path.join(ckpt, '{}_best_checkpoint'.format(ep)))
        torch.save({'salt': torch.tensor(ep)}, os.path.join(ckpt, '{}_best_checkpoint'.format(ep), 'params.pth'))
    np.save(os.path.join(ckpt, 'epoch_ranking.npy'), np.array(EPOCHS))


# ------------------------------------------------------------------------------------------------------------------- one rank
def _install_stand_ins(forwards):
    """the numpy loader ops, the CPU consolidation, and a record of every spatial_tiling_forward call: (pid, checkpoint rank, mirror)"""
    import _loader_cases as LC
    import consolidate_oracle as CO
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import predictor as P
    D.CudaOps = LC.NumpyOps
    P.weighted_box_clustering = CO.weighted_box_clustering
    P.nms_2to3D = CO.nms_2to3D
    tiling = P.Predictor.spatial_tiling_forward

    def recorded(self, batch, patch_crops=None, n_aug='0'):
        forwards.append((batch['pid'], self.rank_ix, n_aug))
        return tiling(self, batch, patch_crops, n_aug)
    P.Predictor.spatial_tiling_forward = recorded


def _net(dim):
    from test_predictor_cpu import StandInNet

    class Net(StandInNet):
        """the stand-in network with a checkpoint: its detections depend on the loaded 'salt'"""
        salt = 0

        def load_state_dict(self, sd):
            assert sd['salt'].device.type == 'cpu'          # map_location: the device of a network without parameters is the CPU
            self.salt = int(sd['salt'])

        def eval(self):
            return self

        def test_forward(self, batch, return_masks=True):
            return StandInNet.test_forward(self, {'data': batch['data'] + 0.01 * self.salt}, return_masks)
    return Net(dim)


def _run(name, root, rank, world, forwards, sharded=True):
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import predictor as P
    cf = _case_cf(name, root)
    cf.fold_dir = os.path.join(root, 'runs', '{}-w{}-r{}{}'.format(name, world, rank, '' if sharded else '-plain'))
    shutil.copytree(os.path.join(root, 'checkpoints'), cf.fold_dir)
    gen = D.get_test_generator(cf, _Log(), rank, world) if sharded else D.get_test_generator(cf, _Log())
    del forwards[:]
    out = P.Predictor(cf, _net(cf.dim), _Log(), 'test').predict_test_set(gen)
    written = sorted(set(os.listdir(cf.fold_dir)) - set(os.listdir(os.path.join(root, 'checkpoints'))))
    raw = None
    if written:
        with open(os.path.join(cf.fold_dir, written[0]), 'rb') as f:
            raw = f.read()
    return {'positions': gen.get('shard_positions'), 'world_size': gen.get('world_size'), 'n_test': gen['n_test'],
            'pids': list(gen['test'].dataset_pids), 'written': written, 'raw': raw, 'results': None if out is None else pickle.dumps(out),
            'forwards': list(forwards)}


def _worker(rank, world, port, root, q):
    try:
        sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
        import torch.distributed as dist
        os.environ['MASTER_ADDR'] = '127.0.0.1'
        os.environ['MASTER_PORT'] = str(port)
        dist.init_process_group('gloo', rank=rank, world_size=world)
        forwards = []
        _install_stand_ins(forwards)
        res = {name: _run(name, root, rank, world, forwards) for name in CASES}
        if world == 1:
            # today's unsharded generator under an initialised process group
            res.update({name + '/plain': _run(name, root, rank, world, forwards, sharded=False) for name in UNCAPPED})
        from medicaldetectiontoolkit_b200 import data_loader as D
        from medicaldetectiontoolkit_b200 import predictor as P
        cf = _case_cf('toy_2d_unpatched_aug', root)
        cf.fold_dir = os.path.join(root, 'checkpoints')
        try:
            P.Predictor(cf, _net(2), _Log(), 'test').predict_test_set(D.get_test_generator(cf, _Log(), rank, world + 1))
            res['mismatch'] = 'no error'
        except RuntimeError as e:
            res['mismatch'] = str(e)
        dist.destroy_process_group()
        q.put((rank, res))
    except BaseException:
        q.put((rank, traceback.format_exc()))


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _spawn_world(world, root):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, root, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=600) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(world):
        assert isinstance(got[r], dict), 'world {} rank {} failed:\n{}'.format(world, r, got[r])
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [got[r] for r in range(world)]


@pytest.fixture(scope='module')
def root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('predict_dist'))
    _write_inputs(root)
    return root


@pytest.fixture(scope='module')
def runs(root):
    return {world: _spawn_world(world, root) for world in WORLDS}


def _capped_pids(name, root):
    """the pids of the first n_test patients, in the order of the unsharded generator"""
    from medicaldetectiontoolkit_b200 import data_loader as D
    cf = _case_cf(name, root)
    data = D.load_dataset(cf, _Log(), None if cf.hold_out_test_set else TEST_IX, pp_data_path=cf.pp_test_data_path)
    n = len(data) if cf.max_test_patients == 'all' else min(cf.max_test_patients, len(data))
    return list(data)[:n]


# ------------------------------------------------------------------------------------------------------------------- checks
@pytest.mark.parametrize('name', list(CASES))
@pytest.mark.parametrize('world', [w for w in WORLDS if w > 1])
def test_rank0_file_and_results_equal_world1(runs, name, world):
    one, r0 = runs[1][0][name], runs[world][0][name]
    assert r0['raw'] is not None and r0['raw'] == one['raw']
    assert r0['results'] is not None and r0['results'] == one['results']
    name_of = 'raw_pred_boxes_hold_out_list.pickle' if CASES[name][1].get('hold_out_test_set', True) else 'raw_pred_boxes_list.pickle'
    assert r0['written'] == one['written'] == [name_of]


@pytest.mark.parametrize('name', UNCAPPED)
def test_world1_equals_the_unsharded_generator(runs, name):
    """the sharded path at world 1 writes the bytes of today's unsharded path, and returns the same results"""
    sharded, plain = runs[1][0][name], runs[1][0][name + '/plain']
    assert plain['raw'] is not None and sharded['raw'] == plain['raw']
    assert sharded['results'] == plain['results']
    assert plain['positions'] is None and plain['world_size'] is None


@pytest.mark.parametrize('name', list(CASES))
def test_shards_partition_the_capped_list(runs, root, name):
    want = _capped_pids(name, root)
    raw = pickle.loads(runs[1][0][name]['raw'])
    assert [pid for _, pid in raw] == want
    for world in WORLDS:
        ranks = [runs[world][r][name] for r in range(world)]
        for r, res in enumerate(ranks):
            assert res['world_size'] == world
            assert res['positions'] == list(range(r, len(want), world)) and res['n_test'] == len(res['positions'])
            assert res['pids'] == [want[p] for p in res['positions']]          # the iterator holds this rank's patients only
        assert sorted(p for res in ranks for p in res['positions']) == list(range(len(want)))


@pytest.mark.parametrize('name', list(CASES))
def test_every_patient_is_forwarded_once_per_checkpoint_and_mirror(runs, root, name):
    mirrors = ['0', '1', '2', '3'] if CASES[name][1]['test_aug'] else ['0']
    want = sorted((pid, str(e), m) for pid in _capped_pids(name, root) for e in range(len(EPOCHS)) for m in mirrors)
    for world in WORLDS:
        assert sorted(f for r in range(world) for f in runs[world][r][name]['forwards']) == want, world


def test_a_world_larger_than_the_test_set_leaves_ranks_empty(runs):
    res = runs[3][2]['lidc_3d_unpatched_capped']
    assert res['n_test'] == 0 and res['positions'] == [] and res['pids'] == [] and res['forwards'] == []
    assert res['results'] is None and res['written'] == []


@pytest.mark.parametrize('world', [w for w in WORLDS if w > 1])
def test_nonzero_ranks_return_none_and_write_nothing(runs, world):
    for r in range(1, world):
        for name in CASES:
            assert runs[world][r][name]['results'] is None and runs[world][r][name]['written'] == [], (r, name)


@pytest.mark.parametrize('world', WORLDS)
def test_a_process_group_of_another_size_raises(runs, world):
    for r in range(world):
        assert 'sharded over {} ranks, but the process group has {}'.format(world + 1, world) in runs[world][r]['mismatch']


def test_bad_rank_or_world_size_raise(root, monkeypatch):
    import _loader_cases as LC
    from medicaldetectiontoolkit_b200 import data_loader as D
    monkeypatch.setattr(D, 'CudaOps', LC.NumpyOps)
    cf = _case_cf('toy_2d_unpatched_aug', root)
    for rank, world in [(2, 2), (-1, 2), (0, 0), (0, None), (None, 2)]:
        with pytest.raises(ValueError):
            D.get_test_generator(cf, _Log(), rank, world)
    gen = D.get_test_generator(cf, _Log(), 1, 2)
    assert gen['shard_positions'] == [1, 3] and gen['world_size'] == 2 and gen['n_test'] == 2


def test_a_sharded_generator_without_a_process_group_raises(root, tmp_path, monkeypatch):
    import torch.distributed as dist
    import _loader_cases as LC
    from medicaldetectiontoolkit_b200 import data_loader as D
    from medicaldetectiontoolkit_b200 import predictor as P
    assert not dist.is_initialized()
    monkeypatch.setattr(D, 'CudaOps', LC.NumpyOps)
    cf = _case_cf('toy_2d_unpatched_aug', root)
    cf.fold_dir = str(tmp_path)
    shutil.copytree(os.path.join(root, 'checkpoints'), cf.fold_dir, dirs_exist_ok=True)
    with pytest.raises(RuntimeError, match='no process group'):
        P.Predictor(cf, _net(2), _Log(), 'test').predict_test_set(D.get_test_generator(cf, _Log(), 0, 1))
    assert sorted(os.listdir(cf.fold_dir)) == sorted(os.listdir(os.path.join(root, 'checkpoints')))
