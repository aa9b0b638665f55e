#!/usr/bin/env python
"""Records what the REFERENCE's UFRCNN+ returns: the unmodified models/ufrcnn.py imported on the CPU through ref_shims.py (nothing is copied),
with the helpers of make_model_golden.py (detweights.fill_, golden_inputs.tame_ with the Mask R-CNN factors, identity torch.randperm,
np.random.seed(0)).

  ufrcnn_model_<case>.npz    whole model, one file per case of CASES: RPN logits and deltas, proposals, second-stage class scores, detections
                             and seg logits (sub-sampled) of a fresh forward; train_forward's detection_target_layer result, every loss term,
                             the SHEM negatives of the RPN loss, box counts and types, the seg_preds sum; parameter gradients (sub-sampled,
                             with norms), the parameters without a gradient and the parameter order; test_forward's detections and seg_preds sum
  ufrcnn_surface.npz         state-dict keys / shapes and a sha256 per tensor of the seeded default initialisation (3D lidc_exp, 2D toy_exp);
                             the make_cf-relevant values of add_mrcnn_configs + the `ufrcnn` block of experiments/{lidc,toy}_exp/configs.py
                             for both dims; get_results on recorded detections with zero-volume and low-confidence rows mixed in

GT boxes are two of the reference's own first-pass proposals per element (as for the Mask R-CNN goldens), so detection_target_layer has
positives; `seg` carries each box's class id inside the box, as the class-specific loader writes it.

Run where the reference tree is present:
  python tests/golden/make_ufrcnn_golden.py [surface] [<case> ...]"""
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import detweights  # noqa: E402
import golden_inputs as GI  # noqa: E402

from medicaldetectiontoolkit_b200.configs import make_cf  # noqa: E402

# name: (dim, patch, batch, exp, overrides, data seed)
CASES = {
    "small": (3, (64, 64, 32), 2, 'lidc_exp', {"post_nms_rois_training": 64, "roi_chunk_size": 1024}, 7),
    "cfg3": (3, (128, 128, 128), 2, 'lidc_exp', {"post_nms_rois_training": 512, "roi_chunk_size": 1024}, 5),
    "2d": (2, (128, 128), 2, 'toy_exp', {}, 5),
}
FINAL_CONV_SCALE = 0.2
N_GRAD_KEYS = 8
N_SUB = 4096          # sub-sampled length of the logits / deltas
N_SUB_GRAD = 2048     # ... and of each recorded gradient
INIT_SEED = 3
INIT_CASES = {"3d": (3, (64, 64, 32), 'lidc_exp'), "2d": (2, (128, 128), 'toy_exp')}
CF_CASES = [('lidc_exp', 3), ('lidc_exp', 2), ('toy_exp', 2)]   # toy_exp has no 3D patch size
# attributes of add_mrcnn_configs + the ufrcnn block that make_cf('ufrcnn') carries (the data-loader / training-loop ones it does not)
CF_KEYS = ["dim", "model", "patch_size", "start_filts", "end_filts", "res_architecture", "norm", "relu", "weight_init", "sixth_pooling",
           "n_latent_dims", "class_specific_seg_flag", "head_classes", "num_seg_classes", "backbone_strides", "rpn_anchor_scales",
           "rpn_anchor_ratios", "rpn_anchor_stride", "pyramid_levels", "n_rpn_features", "rpn_bbox_std_dev", "bbox_std_dev", "window", "scale",
           "rpn_train_anchors_per_image", "train_rois_per_image", "roi_positive_ratio", "anchor_matching_iou", "shem_poolsize", "pool_size",
           "mask_pool_size", "mask_shape", "pre_nms_limit", "rpn_nms_threshold", "roi_chunk_size", "post_nms_rois_training",
           "post_nms_rois_inference", "model_max_instances_per_batch_element", "detection_nms_threshold", "model_min_confidence",
           "operate_stride1", "frcnn_mode", "return_masks_in_val", "return_masks_in_test", "n_plot_rpn_props", "learning_rate",
           "backbone_shapes", "n_anchors_per_pos"]


def case_cf(case):
    dim, patch, B, exp, over, _ = CASES[case]
    cf = make_cf('ufrcnn', dim, patch, exp=exp, batch_size=B)
    for k, v in over.items():
        setattr(cf, k, v)
    return cf


def weights_(net):
    """name-keyed deterministic weights (same keys on the reference's net and ours), heads tamed so that softmaxes are not saturated"""
    GI.tame_(detweights.fill_(net), 'mrcnn')
    with torch.no_grad():
        for name, p in net.named_parameters():
            if name.startswith("final_conv."):
                p.mul_(FINAL_CONV_SCALE)
    return net


def cuboid_batch(cf, data, boxes, labels):
    """batch dict from explicit GT boxes; seg holds each box's class id inside the box (class-specific seg)"""
    B = data.shape[0]
    seg = np.zeros((B, 1) + tuple(cf.patch_size), dtype=np.uint8)
    for b in range(B):
        for bx, lab in zip(boxes[b], labels[b]):
            sl = (slice(int(bx[0]), int(bx[2])), slice(int(bx[1]), int(bx[3]))) + ((slice(int(bx[4]), int(bx[5])),) if cf.dim == 3 else ())
            seg[(b, 0) + sl] = int(lab)
    return {'data': data, 'seg': seg, 'bb_target': [np.asarray(b) for b in boxes], 'roi_labels': [np.asarray(l) for l in labels],
            'pid': ['u%d' % i for i in range(B)]}


def batch_from_golden(cf, g, case):
    """the batch of a recorded case: the seeded image + the recorded GT boxes / labels"""
    dim, patch, B, exp, over, seed = CASES[case]
    data = GI.synthetic_batch(cf, B, seed=seed)['data']
    bt, lab = g["bb_target"], g["roi_labels"]
    boxes = [bt[bt[:, -1] == b][:, :-1].astype(np.int64) for b in range(B)]
    labels = [lab[bt[:, -1] == b] for b in range(B)]
    return cuboid_batch(cf, data, boxes, labels)


def gt_from_proposals(props, dim, B):
    """two of the reference's own first-pass proposals per element (rounded, every extent >= 4 voxels)"""
    boxes, labels = [], []
    for b in range(B):
        p = np.asarray(props[b])
        q = np.round(p[:, :2 * dim])
        ext = np.stack([q[:, 2] - q[:, 0], q[:, 3] - q[:, 1]] + ([q[:, 5] - q[:, 4]] if dim == 3 else []), 1)
        ok = np.where((ext.min(1) >= 4) & (p[:, 2 * dim] > 0))[0]
        pick = ok[[0, len(ok) // 2]] if len(ok) > 1 else ok[:1]
        boxes.append(q[pick].astype(np.int64))
        labels.append(np.array([1 + (i + b) % 2 for i in range(len(pick))]))
    return boxes, labels


def det_rows(boxes, dim):
    """det boxes of a results dict -> rows (element, class, coords..., score)"""
    rows = [[b, d['box_pred_class_id']] + list(np.asarray(d['box_coords'], np.float64)) + [float(d['box_score'])]
            for b, bl in enumerate(boxes) for d in bl if d['box_type'] == 'det']
    return np.array(rows, np.float64).reshape(-1, 2 * dim + 3)


def grad_keys(names, nograd):
    """evenly spaced parameters with a gradient, plus the seg head and the second-stage outputs"""
    cand = [n for n in names if n not in nograd]
    idx = np.linspace(0, len(cand) - 1, N_GRAD_KEYS).round().astype(int)
    extra = ["fpn.P0_conv2.weight", "final_conv.weight", "final_conv.bias", "rpn.conv_class.weight", "classifier.linear_class.weight",
             "classifier.linear_bbox.bias"]
    return sorted(set([cand[i] for i in idx] + extra), key=names.index)


def np_(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def make_model(case):
    import ref_shims as RS
    from make_model_golden import Patched, identity_randperm, recorder
    cf = case_cf(case)
    dim, _, B, _, _, seed = CASES[case]
    RS.install_import_shims()
    out = {}
    t0 = time.time()
    with RS.torch04_semantics(), Patched((torch, "randperm", identity_randperm)):
        m = RS.load_ref_module("ufrcnn")
        net = weights_(m.net(RS.ref_cf(cf), RS.Logger()))
        data = GI.synthetic_batch(cf, B, seed=seed)['data']
        img = torch.from_numpy(data).float()
        with torch.no_grad():
            _, _, props, _, _ = net.forward(img)
        boxes, labels = gt_from_proposals(props, dim, B)
        batch = cuboid_batch(cf, data, boxes, labels)
        out["bb_target"] = np.concatenate([np.concatenate([b, np.full((len(b), 1), i)], 1) for i, b in enumerate(boxes)], 0)
        out["roi_labels"] = np.concatenate(labels)

        log = {}
        patches = [(F, "cross_entropy", recorder(F.cross_entropy, log, "ce")),
                   (m.mutils, "batch_dice", recorder(m.mutils.batch_dice, log, "batch_dice"))]
        for fn in ("compute_rpn_class_loss", "compute_rpn_bbox_loss", "compute_mrcnn_class_loss", "compute_mrcnn_bbox_loss",
                   "detection_target_layer", "refine_detections"):
            patches.append((m, fn, recorder(getattr(m, fn), log, fn)))
        with Patched(*patches):
            np.random.seed(0)
            res = net.train_forward(batch)
            res['torch_loss'].backward()
            np.random.seed(0)
            n_ref = len(log["refine_detections"])
            with torch.no_grad():
                tres = net.test_forward({'data': data})
            out["test_detections"] = np_(log["refine_detections"][n_ref])
        out["test_seg_preds_sum"] = np.array([float(np.asarray(tres['seg_preds']).sum())])
        out["test_det_rows"] = det_rows(tres['boxes'], dim)

        out["loss"] = np_(res['torch_loss']).reshape(-1)
        out["rpn_class_loss"] = np.array([float(np_(l[0]).reshape(-1)[0]) for l in log["compute_rpn_class_loss"]])
        out["rpn_neg_ix"] = np.concatenate([np.asarray(l[1]).astype(np.int64).reshape(-1) for l in log["compute_rpn_class_loss"]])
        out["rpn_bbox_loss"] = np.array([float(np_(l).reshape(-1)[0]) for l in log["compute_rpn_bbox_loss"]])
        out["mrcnn_class_loss"] = np_(log["compute_mrcnn_class_loss"][0]).reshape(-1)
        out["mrcnn_bbox_loss"] = np_(log["compute_mrcnn_bbox_loss"][0]).reshape(-1)
        out["dice"] = np_(log["batch_dice"][-1]).reshape(-1)
        out["seg_ce"] = np_(log["ce"][-1]).reshape(-1)
        six, tcls, tdel = log["detection_target_layer"][0]
        out["dtl_ix"], out["dtl_cls"], out["dtl_deltas"] = np_(six), np_(tcls), np_(tdel)
        out["train_detections"] = np_(log["refine_detections"][0])
        out["n_boxes"] = np.array([len(b) for b in res['boxes']])
        out["box_types"] = np.array(sorted(set(bx['box_type'] for b in res['boxes'] for bx in b)))
        out["seg_preds_sum"] = np.array([float(np.asarray(res['seg_preds']).sum())])
        names = [k for k, _ in net.named_parameters()]
        params = dict(net.named_parameters())
        nograd = [k for k in names if params[k].grad is None]
        keys = grad_keys(names, set(nograd))
        out["grad_keys"] = np.array(keys)
        for k in keys:
            out["grad__" + k] = detweights.subsample(np_(params[k].grad), N_SUB_GRAD)
            out["gradnorm__" + k] = np.array([float(params[k].grad.norm())])
        out["nograd"] = np.array(nograd)
        out["keys"] = np.array(names)
        out["logger_string"] = np.array(res['logger_string'])

        # continuous outputs of a fresh forward (same weights; train_forward does not change them)
        with torch.no_grad():
            rl, rd, pb, det, seg_logits = net.forward(img)
        out["rpn_logits"], out["rpn_deltas"] = detweights.subsample(np_(rl), N_SUB), detweights.subsample(np_(rd), N_SUB)
        out["rpn_logits_shape"] = np.array(rl.shape)
        out["proposals"] = np.asarray(pb)
        out["class_scores"] = np_(net.batch_mrcnn_class_scores)
        out["detections"] = np_(det)
        out["seg_logits"] = detweights.subsample(np_(seg_logits), N_SUB)
        out["seg_logits_shape"] = np.array(seg_logits.shape)
        # margin of the SHEM picks: lowest selected negative vs best unselected negative of the same element (printed; want >> 1e-4)
        fg = out["class_scores"][:, 1:].max(1)
        P_ = fg.shape[0] // B
        neg_ix = out["dtl_ix"][out["dtl_cls"] == 0]
        for b in range(B):
            sel = neg_ix[(neg_ix >= b * P_) & (neg_ix < (b + 1) * P_)]
            rest = np.setdiff1d(np.arange(b * P_, (b + 1) * P_), out["dtl_ix"])
            if sel.size:
                print("    shem margin elem", b, float(fg[sel].min() - np.sort(fg[rest])[-1]), "sel", sel)
    path = os.path.join(HERE, "ufrcnn_model_%s.npz" % case)
    np.savez_compressed(path, **out)
    print(case, res['logger_string'], "| dtl_cls", out["dtl_cls"], "| dets", out["detections"].shape, "test dets", out["test_detections"].shape,
          "| nograd", len(nograd), "| %.1fs" % (time.time() - t0), "->", os.path.getsize(path), "bytes", flush=True)


def _jsonable(v):
    if isinstance(v, np.ndarray):
        return v.tolist()
    if isinstance(v, (np.integer, np.floating)):
        return v.item()
    if isinstance(v, (list, tuple)):
        return [_jsonable(x) for x in v]
    if isinstance(v, dict):
        return {str(k): _jsonable(x) for k, x in v.items()}
    return v


def ref_config(exp, dim):
    """the reference's experiments/<exp>/configs.py with model = 'ufrcnn' and the given dim (both are plain assignments in its __init__:
    a subclass pins them with read-only properties)"""
    import importlib.util
    import ref_shims as RS
    spec = importlib.util.spec_from_file_location("ref_cfg_" + exp, os.path.join(RS.REF, "experiments", exp, "configs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    class Pinned(mod.configs):
        dim = property(lambda self: dim, lambda self, v: None)
        model = property(lambda self: 'ufrcnn', lambda self, v: None)

    c = Pinned(server_env=False)
    return {k: _jsonable(getattr(c, k)) for k in CF_KEYS if hasattr(c, k)}


def make_surface():
    import ref_shims as RS
    RS.install_import_shims()
    out = {}
    with RS.torch04_semantics():
        m = RS.load_ref_module("ufrcnn")
        for tag, (dim, patch, exp) in INIT_CASES.items():
            torch.manual_seed(INIT_SEED)
            net = m.net(RS.ref_cf(make_cf('ufrcnn', dim, patch, exp=exp)), RS.Logger())
            sd = net.state_dict()
            out["init_%s/keys" % tag] = np.array(list(sd.keys()))
            out["init_%s/shapes" % tag] = np.array([",".join(str(s) for s in v.shape) for v in sd.values()])
            out["init_%s/sha256" % tag] = np.array([hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest() for v in sd.values()])
            print("init", tag, len(sd), "tensors")

        # get_results on the recorded detections of the small case, with zero-volume and low-confidence rows mixed in
        g = np.load(os.path.join(HERE, "ufrcnn_model_small.npz"))
        det = g["detections"].astype(np.float32).copy()
        rs = np.random.RandomState(17)
        n = det.shape[0]
        low = rs.permutation(n)[:max(1, n // 3)]
        det[low, -1] = rs.uniform(0.0, 0.2, size=low.size).astype(np.float32)
        det[low[:1], -1] = 0.1                                      # exactly at model_min_confidence: kept (>=)
        flat = rs.permutation(n)[:max(1, n // 5)]
        for i, j in enumerate(flat):
            ax = [(0, 2), (1, 3), (4, 5)][i % 3]
            det[j, ax[1]] = det[j, ax[0]] + (0 if i % 2 == 0 else -1)   # empty or inverted extent
        seg_logits = torch.from_numpy(rs.randn(2, 3, 8, 8, 4).astype(np.float32))
        cf = case_cf("small")
        res = m.get_results(RS.ref_cf(cf), (2, 1, 64, 64, 32), torch.from_numpy(det), seg_logits)
        out["get_results/detections"] = det
        out["get_results/seg_logits"] = seg_logits.numpy()
        out["get_results/rows"] = det_rows(res['boxes'], 3)
        out["get_results/seg_preds"] = np.asarray(res['seg_preds'])
        print("get_results", n, "->", out["get_results/rows"].shape[0], "boxes")
    for exp, dim in CF_CASES:
        out["config/%s/%dd" % (exp, dim)] = np.array(json.dumps(ref_config(exp, dim)))
    path = os.path.join(HERE, "ufrcnn_surface.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(int(os.environ.get("THREADS", "8")))
    what = sys.argv[1:] or list(CASES) + ["surface"]
    for w in what:
        if w == "surface":
            make_surface()
        else:
            make_model(w)
