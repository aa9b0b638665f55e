"""UFRCNN+ without a GPU: the state-dict surface and the seeded default initialisation against the reference's models/ufrcnn.py, make_cf('ufrcnn')
against the reference's experiment configs, get_results on recorded detections, and the data-parallel gradient exchange on a model whose mask.*
and fpn.P1_conv2.* parameters never get a gradient.  The reference side was recorded by tests/golden/make_ufrcnn_golden.py surface."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
import make_ufrcnn_golden as G  # noqa: E402

from medicaldetectiontoolkit_b200 import ufrcnn  # noqa: E402
from medicaldetectiontoolkit_b200.configs import make_cf  # noqa: E402


@pytest.fixture(scope="module")
def surface():
    return np.load(os.path.join(GOLD, "ufrcnn_surface.npz"))


@pytest.mark.parametrize("tag", list(G.INIT_CASES))
def test_state_dict_and_seeded_default_init_equal_the_reference(surface, tag):
    """same keys, shapes and order; under the same seed every tensor is bit-identical (module creation order fpn, rpn, classifier, mask,
    final_conv, and the same RNG use per module)"""
    dim, patch, exp = G.INIT_CASES[tag]
    torch.manual_seed(G.INIT_SEED)
    sd = ufrcnn.net(make_cf('ufrcnn', dim, patch, exp=exp)).state_dict()
    assert list(sd) == list(surface["init_%s/keys" % tag])
    assert [",".join(str(s) for s in v.shape) for v in sd.values()] == list(surface["init_%s/shapes" % tag])
    got = [hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest() for v in sd.values()]
    differ = [k for k, a, b in zip(sd, got, surface["init_%s/sha256" % tag]) if a != b]
    assert not differ, differ


def test_reference_state_dict_loads_key_for_key(surface):
    """a state dict with the reference's keys and shapes loads strictly"""
    net = ufrcnn.net(make_cf('ufrcnn', 3, (64, 64, 32)))
    keys, shapes = list(surface["init_3d/keys"]), list(surface["init_3d/shapes"])
    ref_sd = {k: torch.zeros([int(x) for x in s.split(",") if x]) for k, s in zip(keys, shapes)}
    net.load_state_dict(ref_sd, strict=True)
    assert all(float(v.abs().sum()) == 0 for v in net.state_dict().values())


@pytest.mark.parametrize("exp,dim", G.CF_CASES)
def test_make_cf_equals_reference_config(surface, exp, dim):
    ref = json.loads(str(surface["config/%s/%dd" % (exp, dim)]))
    cf = make_cf('ufrcnn', dim, ref["patch_size"], exp=exp)
    missing = [k for k in ref if not hasattr(cf, k)]
    assert not missing, missing
    differ = {k: (G._jsonable(getattr(cf, k)), v) for k, v in ref.items() if G._jsonable(getattr(cf, k)) != v}
    assert not differ, differ
    # the Mask R-CNN values every other model keeps are untouched
    mr = make_cf('mrcnn', dim, ref["patch_size"], exp=exp)
    assert (mr.operate_stride1, mr.num_seg_classes, mr.frcnn_mode, mr.class_specific_seg_flag) == (False, 2, False, False)
    assert mr.roi_chunk_size == (2500 if dim == 2 else 600) and mr.n_plot_rpn_props == 30 and len(mr.learning_rate) == 100


def test_get_results_matches_reference(surface):
    """zero-volume rows dropped, scores >= model_min_confidence kept, argmax label map: on recorded detections with such rows mixed in"""
    cf = G.case_cf("small")
    det = torch.from_numpy(surface["get_results/detections"])
    seg_logits = torch.from_numpy(surface["get_results/seg_logits"])
    res = ufrcnn.get_results(cf, (2, 1, 64, 64, 32), det, seg_logits)
    rows = G.det_rows(res['boxes'], 3)
    want = surface["get_results/rows"]
    assert rows.shape == want.shape and 0 < rows.shape[0] < det.shape[0]
    np.testing.assert_array_equal(rows, want)
    assert all(d['box_coords'].dtype == np.int32 for bl in res['boxes'] for d in bl)
    assert res['seg_preds'].dtype == np.uint8
    np.testing.assert_array_equal(res['seg_preds'], surface["get_results/seg_preds"])


# ------------------------------------------------------------------------------------------------------------------ data parallel
def _never_grad(name):
    return name.startswith("mask.") or name.startswith("fpn.P1_conv2.")


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    from medicaldetectiontoolkit_b200 import ufrcnn as U
    from medicaldetectiontoolkit_b200.configs import make_cf as mk
    from medicaldetectiontoolkit_b200.parallel import FlatGradAllReduce
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)   # identical replicas
    net = U.net(mk('ufrcnn', 3, (64, 64, 32)))
    red = FlatGradAllReduce(net, world)
    red.zero_grad()
    # a step's gradient pattern: every parameter but mask.* and fpn.P1_conv2.* gets the gradient (rank + 1) * (i % 7 + 1), those get none
    used = [(n, p) for n, p in net.named_parameters() if not _never_grad(n)]
    sum(((rank + 1) * (i % 7 + 1) * p).sum() for i, (n, p) in enumerate(used)).backward()
    local_sum = float(red.flat.double().sum())
    red.all_reduce()
    # the full buffers are too large to ship back: check them here against the known mean, (1 + 2) / 2 * (i % 7 + 1)
    scale = {n: 1.5 * (i % 7 + 1) for i, (n, _) in enumerate(used)}
    res, off = {}, 0
    for n, p in net.named_parameters():
        seg = red.flat[off:off + p.numel()]
        want = scale.get(n, 0.0)
        res[n] = (bool(torch.all(seg == want)), p.grad.data_ptr() == seg.data_ptr())
        off += p.numel()
    q.put((rank, local_sum, res))
    dist.destroy_process_group()


def _free_port():
    import socket
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_flat_grad_allreduce_with_never_grad_parameters():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = sorted([q.get(timeout=300) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    never = [n for n in out[0][2] if _never_grad(n)]
    assert any(n.startswith("mask.") for n in never) and any(n.startswith("fpn.P1_conv2.") for n in never)
    for rank, local_sum, res in out:
        bad = [n for n, (ok, view) in res.items() if not (ok and view)]
        assert not bad, (rank, bad)          # averaged gradients everywhere, zeros for the never-grad parameters, .grad views of the buffer
    assert out[1][1] == 2 * out[0][1] != 0   # ranks really had different local gradients
