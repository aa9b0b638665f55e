"""UFRCNN+ on the GPU against the unmodified models/ufrcnn.py (tests/golden/make_ufrcnn_golden.py): RPN outputs, seg logits, proposals,
detections, detection targets, every loss term, SHEM negatives and parameter gradients, test_forward, the Predictor in test mode and a
reproducible train step.  Tolerances are those of the Mask R-CNN and Retina U-Net whole-model tests (tests/test_model_golden.py)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLD)
import detweights  # noqa: E402
import make_ufrcnn_golden as G  # noqa: E402

from medicaldetectiontoolkit_b200 import model_utils as mutils, native_ops, ufrcnn as UF  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
sub = detweights.subsample
LOSS_FNS = ("compute_rpn_class_loss", "compute_rpn_bbox_loss", "compute_mrcnn_class_loss", "compute_mrcnn_bbox_loss", "detection_target_layer")


@pytest.fixture(autouse=True)
def identity_sampling():
    old = mutils.SAMPLING
    mutils.SAMPLING = "identity"
    yield
    mutils.SAMPLING = old


def _np(x):
    return x.detach().cpu().numpy()


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)) if a.size else 0.0


def _rel_l2(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _match_fraction(got, want, dim):
    """fraction of the reference's detections found in ours (same rounded box, element, class; score within 1e-4)"""
    if want.shape[0] == 0:
        return 1.0
    hit = 0
    for w in want:
        same = np.all(got[:, :2 * dim + 2] == w[:2 * dim + 2], axis=1) & (np.abs(got[:, -1] - w[-1]) <= 1e-4)
        hit += bool(same.any())
    return hit / want.shape[0]


def _build(case):
    g = np.load(os.path.join(GOLD, "ufrcnn_model_%s.npz" % case))
    cf = G.case_cf(case)
    net = G.weights_(UF.net(cf)).to(DEV)
    return g, cf, net, G.batch_from_golden(cf, g, case)


class _Recorder:
    """records the results of the module-level loss / sampling functions of ufrcnn.py and of the fused seg loss during a train step"""

    def __init__(self):
        self.log = {}
        self.orig = {n: getattr(UF, n) for n in LOSS_FNS}
        self.orig_seg = native_ops.seg_loss

    def _wrap(self, n, fn):
        def f(*a, **k):
            out = fn(*a, **k)
            self.log.setdefault(n, []).append(out)
            return out
        return f

    def __enter__(self):
        for n in LOSS_FNS:
            setattr(UF, n, self._wrap(n, self.orig[n]))
        native_ops.seg_loss = self._wrap("seg_loss", self.orig_seg)
        return self.log

    def __exit__(self, *a):
        for n in LOSS_FNS:
            setattr(UF, n, self.orig[n])
        native_ops.seg_loss = self.orig_seg


def _check_grads(net, g, tol=1e-2):
    params = dict(net.named_parameters())
    assert list(params) == list(g["keys"])                                          # the reference's parameters, in order
    nograd = sorted(k for k, p in params.items() if p.grad is None)
    assert nograd == sorted(g["nograd"])
    assert any(k.startswith("mask.") for k in nograd) and "fpn.P1_conv2.weight" in nograd
    errs = {}
    for k in g["grad_keys"]:
        a, b = sub(_np(params[k].grad), G.N_SUB_GRAD).astype(np.float64), g["grad__" + k].astype(np.float64)
        errs[k] = _rel_l2(a, b)
        nrm, want = float(params[k].grad.norm()), float(g["gradnorm__" + k][0])
        assert abs(nrm - want) <= tol * want, (k, nrm, want)
        if want > 0:
            assert float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-300)) >= 1 - tol * tol, k      # same direction
        else:
            assert nrm == 0, k           # a pyramid level that no sampled anchor or roi lies on: no gradient in the reference either
    assert max(errs.values()) <= tol, errs


@pytest.mark.parametrize("case", list(G.CASES))
def test_ufrcnn_vs_reference(case):
    g, cf, net, batch = _build(case)
    img = torch.from_numpy(batch['data']).to(DEV)
    with torch.no_grad():
        rl, rd, props, det, seg = net.forward(img)
    assert list(rl.shape) == g["rpn_logits_shape"].tolist() and list(seg.shape) == g["seg_logits_shape"].tolist()
    assert _rel(sub(_np(rl), G.N_SUB), g["rpn_logits"]) <= 1e-4
    assert _rel(sub(_np(rd), G.N_SUB), g["rpn_deltas"]) <= 1e-4
    assert _rel(sub(_np(seg), G.N_SUB), g["seg_logits"]) <= 1e-4
    p_got, p_want = _np(props), g["proposals"]
    assert p_got.shape == p_want.shape
    close = np.all(np.abs(p_got - p_want) <= 1e-3 * np.maximum(1.0, np.abs(p_want)), axis=2)
    assert close.mean() >= 0.95, close.mean()
    rows = close.reshape(-1)
    assert _rel(_np(net.batch_mrcnn_class_scores)[rows], g["class_scores"][rows]) <= 1e-4
    assert _match_fraction(_np(det), g["detections"], cf.dim) >= 0.9

    with _Recorder() as log:
        np.random.seed(0)
        res = net.train_forward(batch)
    res['torch_loss'].backward()
    six, tcls, tdel = log["detection_target_layer"][0]
    assert _np(tcls).tolist() == g["dtl_cls"].tolist()
    got_ix, want_ix = _np(six), g["dtl_ix"]
    n_pos = int((g["dtl_cls"] > 0).sum())
    assert n_pos > 0 and got_ix[:n_pos].tolist() == want_ix[:n_pos].tolist()              # positive samples: exact
    if got_ix.tolist() != want_ix.tolist():
        # SHEM negatives are the top-scoring ones: a pick may differ from the reference's only where the reference scores are a near-tie
        ref_fg = g["class_scores"][:, 1:].max(1)
        P = ref_fg.shape[0] // len(batch['data'])
        assert sorted(got_ix[n_pos:] // P) == sorted(want_ix[n_pos:] // P)
        assert np.all(ref_fg[got_ix[n_pos:]] >= ref_fg[want_ix[n_pos:]].min() - 1e-4), (got_ix, want_ix)
        pytest.skip("SHEM near-tie resolved differently than the reference (scores within 1e-4): sample-dependent losses not comparable")
    assert _rel(_np(tdel), g["dtl_deltas"]) <= 1e-3
    dice, ce = log["seg_loss"][0]
    got = {
        "rpn_class_loss": np.array([float(l[0]) for l in log["compute_rpn_class_loss"]]),
        "rpn_bbox_loss": np.array([float(l) for l in log["compute_rpn_bbox_loss"]]),
        "mrcnn_class_loss": np.array([float(log["compute_mrcnn_class_loss"][0])]),
        "mrcnn_bbox_loss": np.array([float(log["compute_mrcnn_bbox_loss"][0])]),
        "dice": np.array([float(dice)]),
        "seg_ce": np.array([float(ce)]),
        "loss": np.array([float(res['torch_loss'])]),
    }
    for k, v in got.items():
        assert np.abs(v - g[k]).max() <= 2e-4 * max(1.0, np.abs(g[k]).max()), (k, v, g[k])
    negs = np.concatenate([_np(l[1])[_np(l[1]) >= 0] for l in log["compute_rpn_class_loss"]])
    assert negs.tolist() == g["rpn_neg_ix"].tolist()
    assert sorted(set(bx['box_type'] for b in res['boxes'] for bx in b)) == list(g["box_types"])
    assert res['seg_preds'].dtype == np.uint8 and res['seg_preds'].shape == (len(batch['data']), 1) + tuple(cf.patch_size)
    assert abs(float(res['seg_preds'].sum()) - g["seg_preds_sum"][0]) <= 1e-4 * res['seg_preds'].size
    assert res['logger_string'].startswith("loss: ") and ", dice_loss: " in res['logger_string']
    assert set(res['monitor_values']) == {'loss', 'class_loss'}
    _check_grads(net, g)


@pytest.mark.parametrize("case", list(G.CASES))
def test_test_forward_vs_reference(case):
    """test_forward uses post_nms_rois_training proposals, as the reference's does; its detections and label map match the reference's"""
    g, cf, net, batch = _build(case)
    res = net.test_forward({'data': batch['data']}, return_masks=True)
    assert net.rpn_rois_batch_info.shape[0] == len(batch['data']) * cf.post_nms_rois_training
    assert all(d['box_type'] == 'det' for bl in res['boxes'] for d in bl)
    assert _match_fraction(G.det_rows(res['boxes'], cf.dim)[:, [*range(2, 2 + 2 * cf.dim), 0, 1, 2 + 2 * cf.dim]],
                           g["test_det_rows"][:, [*range(2, 2 + 2 * cf.dim), 0, 1, 2 + 2 * cf.dim]], cf.dim) >= 0.9
    assert res['seg_preds'].dtype == np.uint8
    assert abs(float(res['seg_preds'].sum()) - g["test_seg_preds_sum"][0]) <= 1e-4 * res['seg_preds'].size


def test_predictor_test_mode(tmp_path):
    """the Predictor calls test_forward(batch, return_masks=...) on every patch of a 3D patient"""
    from medicaldetectiontoolkit_b200 import predictor
    cf = G.case_cf("small")
    for k, v in dict(test_aug=False, merge_2D_to_3D_preds=False, merge_3D_iou=0.1, return_masks_in_test=False, wcs_iou=1e-5, fold_dir=str(tmp_path),
                     fold=0, test_n_epochs=1, hold_out_test_set=False, folds=[0], exp_dir=str(tmp_path), model_min_confidence=0.0).items():
        setattr(cf, k, v)
    torch.manual_seed(0)
    net = G.weights_(UF.net(cf)).to(DEV)
    net.eval()
    np.save(os.path.join(str(tmp_path), 'epoch_ranking.npy'), np.array([1]))
    vol = np.random.RandomState(6).rand(1, 1, 96, 64, 32).astype(np.float32)
    crops = [[0, 64, 0, 64, 0, 32], [32, 96, 0, 64, 0, 32]]
    patient = {'data': np.stack([vol[0, :, c[0]:c[1]] for c in crops]), 'patch_crop_coords': crops, 'original_img_shape': vol.shape, 'pid': 'p0',
               'patient_bb_target': np.array([[[5, 5, 20, 20, 2, 9]]]), 'patient_roi_labels': np.array([[1]])}
    out = predictor.Predictor(cf, net, _Log(), 'test').predict_patient(patient)
    dets = [d for bl in out['boxes'] for d in bl if d['box_type'] == 'det']
    assert dets and all(d['box_pred_class_id'] in (1, 2) for d in dets)


class _Log:
    def info(self, *a, **k):
        pass


def test_train_step_reproducible():
    """two train steps from the same weights and batch: every loss term, the detections and the gradients of final_conv.*, rpn.* and
    classifier.* are bit-identical.  The fpn.* gradients receive the RoIAlign backward's float-atomic scatter, whose summation order varies
    from run to run: they agree to relative L2 1e-5 (measured on an H100 80GB HBM3 at 700 W: at most 2.0e-6, at fpn.C0.0.0.weight)"""
    mutils.SAMPLING = "random"
    cf = G.case_cf("small")
    torch.manual_seed(0)
    net = G.weights_(UF.net(cf)).to(DEV)
    g = np.load(os.path.join(GOLD, "ufrcnn_model_small.npz"))
    batch = G.batch_from_golden(cf, g, "small")

    def step():
        torch.manual_seed(1)
        np.random.seed(1)
        net.zero_grad(set_to_none=True)
        with _Recorder() as log:
            res = net.train_forward(batch)
        res['torch_loss'].backward()
        terms = [float(l[0]) for l in log["compute_rpn_class_loss"]] + [float(l) for l in log["compute_rpn_bbox_loss"]] + \
            [float(log["compute_mrcnn_class_loss"][0]), float(log["compute_mrcnn_bbox_loss"][0])] + [float(x) for x in log["seg_loss"][0]] + \
            [float(res['torch_loss'])]
        dets = [[(d['box_pred_class_id'], d['box_coords'].tolist(), float(d['box_score'])) for d in bl if d['box_type'] == 'det'] for bl in res['boxes']]
        grads = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
        return terms, dets, grads, res['seg_preds']

    t1, d1, g1, s1 = step()
    t2, d2, g2, s2 = step()
    assert t1 == t2 and d1 == d2 and np.array_equal(s1, s2)
    assert sorted(g1) == sorted(g2)
    exact = [k for k in g1 if k.split(".")[0] in ("final_conv", "rpn", "classifier")]
    assert any(k.startswith("final_conv.") for k in exact) and any(k.startswith("classifier.") for k in exact)
    differ = [k for k in exact if not torch.equal(g1[k], g2[k])]
    assert not differ, differ
    for k in g1:
        if k.startswith("fpn."):
            assert _rel_l2(_np(g1[k]), _np(g2[k])) <= 1e-5, k
