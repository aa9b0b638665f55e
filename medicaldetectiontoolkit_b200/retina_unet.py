"""Retina U-Net (one-stage detector + full-resolution segmentation head) on libmdt_b200 — the operator surface of the reference's
models/retina_unet.py (`net(cf, logger)` with `train_forward(batch)`, `test_forward(batch)`, `forward(img)` and the same
results_dict keys), re-designed so that a training step never leaves the GPU:

  reference (file:line)                                         here
  ------------------------------------------------------------  ------------------------------------------------------------------
  Classifier / BBRegressor towers      retina_unet.py:40-119    same modules/keys, tensor-core convs, logits stay channels-last (no permute copy)
  numpy gt_anchor_matching per element retina_unet.py:416       fp64 device kernels (csrc/anchor_match.cu) through model_utils
  compute_class_loss / shem            :126-164, mutils :674    fixed-shape top-k formulation, no nonzero()/host sync
  refine_detections                    :194-271                 top-k instead of a 5.4 M-element sort; ONE batched multi-class NMS launch
  nms_3D per (batch, class) + D2H mask pth_nms.py / nms_cuda.c  csrc/nms.cu bitmask + on-device reduction
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import model_utils as mutils
from . import native_ops
from ._detector import Detector, anchor_losses, append_anchor_boxes, match_anchors, seg_loss_terms
from .backbone import FPN
from .conv import NDConvGenerator, no_split_consumer

_CL3 = torch.channels_last_3d


# ------------------------------------------------------------------------------------------------------------------ heads
class _Tower(nn.Module):
    """4 x (conv3 + ReLU) + conv3 -> [b, n_anchors, out_per_anchor]; shared across pyramid levels"""

    def __init__(self, cf, conv, out_per_anchor):
        super().__init__()
        self.dim = conv.dim
        self.out_per_anchor = out_per_anchor
        n_in, n_feat, s = cf.end_filts, cf.n_rpn_features, cf.rpn_anchor_stride
        self.conv_1 = conv(n_in, n_feat, ks=3, stride=s, pad=1, relu=cf.relu)
        self.conv_2 = conv(n_feat, n_feat, ks=3, stride=s, pad=1, relu=cf.relu)
        self.conv_3 = conv(n_feat, n_feat, ks=3, stride=s, pad=1, relu=cf.relu)
        self.conv_4 = conv(n_feat, n_feat, ks=3, stride=s, pad=1, relu=cf.relu)
        self.conv_final = no_split_consumer(conv(n_feat, cf.n_anchors_per_pos * out_per_anchor, ks=3, stride=s, pad=1, relu=None))

    def forward(self, x):
        y = self.conv_final(self.conv_4(self.conv_3(self.conv_2(self.conv_1(x)))))
        axes = (0, 2, 3, 1) if self.dim == 2 else (0, 2, 3, 4, 1)
        # channels-last memory == the permuted layout the reference materialises with .permute().contiguous() (retina_unet.py:71-75)
        y = y.permute(*axes).contiguous()
        return [y.view(x.size(0), -1, self.out_per_anchor)]


class Classifier(_Tower):
    """class logits (b, n_anchors, n_classes)   (retina_unet.py:40-78)"""

    def __init__(self, cf, conv):
        super().__init__(cf, conv, cf.head_classes)
        self.n_classes = cf.head_classes


class BBRegressor(_Tower):
    """box deltas (b, n_anchors, 2*dim)   (retina_unet.py:82-119)"""

    def __init__(self, cf, conv):
        super().__init__(cf, conv, conv.dim * 2)


# ------------------------------------------------------------------------------------------------------------------ losses
FUSED_LOSSES = True   # False: the formulation in torch ops (kept as the in-repo cross-check of the fused kernels, tests/test_model_gpu.py)


def _topk_long(score, k, blk=8192):
    """exact sorted top-k of a long 1-D tensor for small k: per-block top-k (one batched launch) + top-k of the nb*k candidates.  The
    library's multi-block radix select costs ~11 launches (0.4 ms) per call on the 1.35 M anchor scores of cfg2; the top-k overall is a
    subset of the per-block top-k, so the result is the same set (ties at the k-th value are arbitrary in both)."""
    A = score.shape[0]
    if A <= 4 * blk or k > 256 or k > blk:
        return torch.topk(score, k, sorted=True)
    nb = (A + blk - 1) // blk
    s2 = F.pad(score, (0, nb * blk - A), value=float('-inf')).view(nb, blk)
    v, i = torch.topk(s2, k, dim=1, sorted=False)
    i = i + torch.arange(nb, device=score.device).unsqueeze(1) * blk
    vv, j = torch.topk(v.reshape(-1), k, sorted=True)
    return vv, i.reshape(-1)[j]


def _positive_indices(anchor_matches, k_pos, pos_ids):
    """first k_pos positive anchor indices in ascending order, padded with A.  pos_ids: the matching's own list of positives (already on
    the device, exact length) — saves a radix top-k over the whole anchor array (1.35 M entries at cfg2) per loss call"""
    A = anchor_matches.shape[0]
    if pos_ids is not None:
        pad = pos_ids.new_full((k_pos,), A)
        n = min(int(pos_ids.shape[0]), k_pos)
        pad[:n] = pos_ids[:n]
        return pad
    idx = torch.arange(A, device=anchor_matches.device)
    return torch.topk(torch.where(anchor_matches > 0, idx, idx.new_full((), A)), k_pos, largest=False, sorted=True)[0]


def compute_class_loss(anchor_matches, class_pred_logits, shem_poolsize=20, max_pos=None, generator=None, pos_ids=None):
    """CE on positive anchors + CE on stochastically-hard-mined negatives (retina_unet.py:126-164, model_utils.py:674-691).

    Fixed-shape, sync-free: positives (at most max_pos) and the SHEM pool (shem_poolsize * n_neg best-scoring negatives) are selected
    with top-k + validity masks instead of nonzero().  Returns (loss, neg_anchor_ix) with neg_anchor_ix = indices INTO THE NEGATIVE
    SUBSET like the reference (int64 CUDA tensor padded with -1).
    """
    A = anchor_matches.shape[0]
    dev = class_pred_logits.device
    if pos_ids is not None and max_pos is not None and FUSED_LOSSES:
        k_pos = int(min(A, max_pos))
        k_pool = int(min(A, shem_poolsize * k_pos))
        if native_ops.shem_supported(class_pred_logits, k_pos, k_pool):
            # one fused selection + loss (csrc/loss_ops.cu): same pool, same uniform keys, same sample as the formulation below
            keys = mutils.rand_keys(k_pool, dev, generator)
            return native_ops.shem_class_loss(class_pred_logits, anchor_matches, pos_ids, keys, k_pos, k_pool, int(min(k_pool, k_pos)), shem_poolsize)
    pos_flag = (anchor_matches > 0)
    n_pos = pos_flag.sum()
    # max_pos is the caller's guarantee on the number of positives (the matching caps it at rpn_train_anchors_per_image // 2); without
    # it the bound is read back from the device (one sync) so that the reference's signature stays lossless for any number of positives
    k_pos = int(min(A, max_pos)) if max_pos is not None else max(1, int(n_pos.item()))
    # first k_pos positive indices in ascending order (stable)
    pos_idx = _positive_indices(anchor_matches, k_pos, pos_ids)
    pos_valid = pos_idx < A
    pos_idx_c = pos_idx.clamp_max(A - 1)
    ce_pos = F.cross_entropy(class_pred_logits[pos_idx_c], anchor_matches[pos_idx_c].clamp_min(0).long(), reduction='none')
    pos_loss = (ce_pos * pos_valid).sum() / pos_valid.sum().clamp_min(1)

    neg_flag = (anchor_matches == -1)
    n_neg_total = neg_flag.sum()
    negative_count = n_pos.clamp_min(1)                                    # np.max((1, n_pos))
    # hardest negatives by max foreground probability (softmax over ALL anchors is one streaming pass; masked afterwards)
    probs = F.softmax(class_pred_logits.detach(), dim=1)
    score = torch.where(neg_flag, probs[:, 1:].max(1)[0], probs.new_full((), -1.0))
    k_pool = int(min(A, shem_poolsize * k_pos))
    pool_score, pool_idx = _topk_long(score, k_pool)
    pool_size = torch.minimum(shem_poolsize * negative_count, n_neg_total)   # model_utils.py:687
    in_pool = (torch.arange(k_pool, device=dev) < pool_size) & (pool_score >= 0)
    # sample `negative_count` of the pool without replacement: smallest random keys among pool members (== randperm(pool)[:n])
    keys = mutils.rand_keys(k_pool, dev, generator)
    keys = torch.where(in_pool, keys, keys.new_full((), 2.0))
    k_neg = int(min(k_pool, k_pos))
    sel_key, sel = torch.topk(keys, k_neg, largest=False)
    neg_valid = (torch.arange(k_neg, device=dev) < negative_count) & (sel_key < 1.5)
    neg_idx = pool_idx[sel]
    ce_neg = F.cross_entropy(class_pred_logits[neg_idx], torch.zeros(k_neg, dtype=torch.long, device=dev), reduction='none')
    neg_loss = (ce_neg * neg_valid).sum() / neg_valid.sum().clamp_min(1)
    # position of each sampled negative inside the negative subset (the reference indexes roi_logits_neg)
    neg_rank = torch.cumsum(neg_flag.long(), 0) - 1
    neg_ix = torch.where(neg_valid, neg_rank[neg_idx], neg_rank.new_full((), -1))
    return (pos_loss + neg_loss) / 2, neg_ix


def compute_bbox_loss(target_deltas, pred_deltas, anchor_matches, max_pos=None, pos_ids=None):
    """smooth-L1 between the predicted deltas of the positive anchors (ascending anchor order) and their targets (retina_unet.py:167-187)"""
    A = anchor_matches.shape[0]
    dev = pred_deltas.device
    k_pos = int(min(A, target_deltas.shape[0] if max_pos is None else max_pos))
    pos_idx = _positive_indices(anchor_matches, k_pos, pos_ids)
    valid = (pos_idx < A)
    pred = pred_deltas[pos_idx.clamp_max(A - 1)]
    l = F.smooth_l1_loss(pred, target_deltas[:k_pos].to(pred.dtype), reduction='none').sum(1)
    n = valid.sum()
    return (l * valid).sum() / (n.clamp_min(1) * pred.shape[1])   # mean over n_pos x 2*dim elements; 0 if no positive


# ------------------------------------------------------------------------------------------------------------------ detections
def refine_detections(anchors, probs, deltas, batch_ixs, cf):
    """anchors (n_anchors, 2*dim); probs (b*n_anchors, n_classes); deltas (b*n_anchors, 2*dim); batch_ixs (b*n_anchors)
    -> (n_det, (y1, x1, y2, x2, (z1), (z2), batch_ix, class_id, score)), at most model_max_instances_per_batch_element per element.

    Same selection as retina_unet.py:194-271 (top pre_nms_limit foreground scores over the whole batch, decode, clip, round, NMS per
    (batch element, class), top-k per element) but as ONE NMS launch: boxes of different (element, class) groups are translated apart
    along y so they can never overlap; the coordinates are rounded pixels, so the IoUs inside a group are bit-identical.
    """
    dim = cf.dim
    n_anchors = anchors.shape[0]
    fg = probs[:, 1:]
    n_fg = fg.shape[1]
    k = int(min(cf.pre_nms_limit, fg.numel()))
    scores, flat_ix = torch.topk(fg.reshape(-1), k, sorted=True)
    row = torch.div(flat_ix, n_fg, rounding_mode='floor')                # torch-0.4 integer `/` (retina_unet.py:212)
    class_ids = flat_ix - row * n_fg + 1
    b_ix = batch_ixs[row]
    pre_anchors = anchors[row % n_anchors]                                 # anchors.repeat(batch, 1)[row]
    std_dev = torch.as_tensor(np.reshape(cf.rpn_bbox_std_dev, [1, dim * 2]), dtype=torch.float32, device=probs.device)
    scale = torch.as_tensor(np.asarray(cf.scale), dtype=torch.float32, device=probs.device)
    apply = mutils.apply_box_deltas_2D if dim == 2 else mutils.apply_box_deltas_3D
    rois = apply(pre_anchors / scale, deltas[row] * std_dev) * scale
    rois = torch.round(mutils.clip_to_window(cf.window, rois))

    # batched multi-class NMS: translate each (batch, class) group to its own y band
    n_groups_cls = n_fg + 1
    band = float(max(cf.window[2], cf.window[3]) + 2)
    offs = (b_ix * n_groups_cls + class_ids).to(rois.dtype) * band
    shifted = rois.clone()
    shifted[:, 0] += offs
    shifted[:, 2] += offs
    dets = torch.cat((shifted, scores.unsqueeze(1)), dim=1)               # already sorted by descending score
    # group-major order (stable: descending score inside every group): greedy NMS of disjoint groups is the union of the per-group runs, and
    # the mask kernel skips every 64x64 tile whose boxes lie in different y bands (csrc/nms.cu: nms_tile_bounds_kernel) - 3/4 of the pair tests
    # with 2 elements x 2 classes
    order_g = torch.sort(b_ix * n_groups_cls + class_ids, stable=True)[1]
    keep_pad, num = native_ops.nms_sorted(dets[order_g].contiguous(), cf.detection_nms_threshold, dim)
    kept_g = torch.zeros(k, dtype=torch.bool, device=probs.device)
    pos = torch.arange(k, device=probs.device)
    valid = pos < num.to(torch.long)
    kept_g[keep_pad.clamp(0, k - 1)[valid]] = True
    kept = torch.empty_like(kept_g)
    kept[order_g] = kept_g                                                # back to descending-score positions
    # top model_max_instances_per_batch_element per element, in score order
    n_b = int(batch_ixs.max().item()) + 1 if batch_ixs.numel() else 1
    onehot = (b_ix.unsqueeze(0) == torch.arange(n_b, device=probs.device).unsqueeze(1)) & kept.unsqueeze(0)   # [n_b, k]: scan along the contiguous dim
    rank = torch.cumsum(onehot.to(torch.int32), 1)
    within = (rank * onehot).sum(0)
    final = kept & (within <= cf.model_max_instances_per_batch_element)
    sel = torch.nonzero(final).squeeze(1)                                  # variable-length result: the one sync of the forward
    return torch.cat((rois[sel], b_ix[sel].unsqueeze(1).float(), class_ids[sel].unsqueeze(1).float(), scores[sel].unsqueeze(1)), dim=1)


def get_results(cf, img_shape, detections, seg_logits, box_results_list=None, host=None):
    """results_dict {'boxes': per-element lists of box dicts, 'seg_preds': uint8 label map} — retina_unet.py:275-333.
    host: optional (detections, seg_preds) numpy arrays already copied to the host (train_forward batches its device->host copies)"""
    det = detections.detach().cpu().numpy() if host is None else host[0]
    dim = cf.dim
    if box_results_list is None:
        box_results_list = [[] for _ in range(img_shape[0])]
    for ix in range(img_shape[0]):
        d = det[det[:, 2 * dim] == ix]
        if d.shape[0] == 0:
            continue
        boxes = d[:, :2 * dim].astype(np.int32)
        class_ids = d[:, 2 * dim + 1].astype(np.int32)
        scores = d[:, 2 * dim + 2]
        vol = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
        if dim == 3:
            vol = vol * (boxes[:, 5] - boxes[:, 4])
        ok = (vol > 0) & (scores >= cf.model_min_confidence)            # drop zero-volume boxes, keep confident ones
        for b, s, c in zip(boxes[ok], scores[ok], class_ids[ok]):
            box_results_list[ix].append({'box_coords': b, 'box_score': s, 'box_type': 'det', 'box_pred_class_id': c})
    results = {'boxes': box_results_list}
    if seg_logits is None:
        results['seg_preds'] = np.zeros(img_shape)[:, 0][:, np.newaxis]
    elif host is not None:
        results['seg_preds'] = host[1]
    else:
        results['seg_preds'] = seg_logits.detach().argmax(1, keepdim=True).to(torch.uint8).cpu().numpy()  # argmax(softmax) == argmax(logits)
    return results


# ------------------------------------------------------------------------------------------------------------------ net
class net(Detector):
    """Retina U-Net.  `operate_stride1`/seg head follow cf (set cf.operate_stride1 False and num_seg_classes 0 for plain RetinaNet)."""

    has_seg_head = True

    def build(self):
        cf = self.cf
        self._check_patch_size()
        conv = NDConvGenerator(cf.dim)
        self._register_anchors()
        self.Fpn = FPN(cf, conv, operate_stride1=cf.operate_stride1)
        self.Classifier = Classifier(cf, conv)
        self.BBRegressor = BBRegressor(cf, conv)
        if self.has_seg_head:
            self.final_conv = no_split_consumer(conv(cf.end_filts, cf.num_seg_classes, ks=1, pad=0, norm=None, relu=None))

    # -------------------------------------------------------------------------------------------------------------- forward
    def forward(self, img):
        """img (b, c, y, x, (z)) -> detections, class_logits (b, n_anchors, n_cls), bb_outputs (b, n_anchors, 2*dim), seg_logits"""
        class_logits, bb_outputs, seg_logits = self._forward_logits(img)
        return self._detect(class_logits, bb_outputs), class_logits, bb_outputs, seg_logits

    def _forward_logits(self, img):
        """the differentiable part of forward(): backbone + heads"""
        fpn_outs = self.Fpn(img)
        if self.has_seg_head:
            seg_logits = self.final_conv(fpn_outs[0])
            first = 1
        else:
            seg_logits = None
            first = 1 if self.cf.operate_stride1 else 0
        fmaps = [fpn_outs[i + first] for i in self.cf.pyramid_levels]
        class_logits = torch.cat([self.Classifier(p)[0] for p in fmaps], dim=1)
        bb_outputs = torch.cat([self.BBRegressor(p)[0] for p in fmaps], dim=1)
        return class_logits, bb_outputs, seg_logits

    def _detect(self, class_logits, bb_outputs):
        """softmax + refine_detections (ends in the one host sync of the forward: a variable-length result)"""
        b, a = class_logits.shape[0], class_logits.shape[1]
        with torch.no_grad():
            batch_ixs = torch.arange(b, device=class_logits.device).unsqueeze(1).repeat(1, a).view(-1)
            flat_softmax = F.softmax(class_logits.detach().view(-1, class_logits.shape[-1]), 1)
            return refine_detections(self.anchors, flat_softmax, bb_outputs.detach().view(-1, bb_outputs.shape[-1]), batch_ixs, self.cf)

    def train_forward(self, batch, **kwargs):
        """batch: {'data', 'seg', 'bb_target', 'roi_labels', ...} numpy -> results_dict with 'torch_loss', 'boxes', 'seg_preds',
        'monitor_values', 'logger_string' (retina_unet.py:381-456).

        Order of work (results are the reference's; the ORDER keeps the GPU queue full): the anchor matching needs only the GT boxes, so it
        (and its host synchronisation) runs first; backbone, heads and all losses are then queued without a sync; the detections for the
        monitoring output (NMS, variable-length result) and every device->host copy come last and share one synchronisation."""
        cf = self.cf
        img = self._to_device(batch['data'])
        box_results_list = [[] for _ in range(img.shape[0])]
        seg = self._seg_to_device(batch['seg'], FUSED_LOSSES) if self.has_seg_head else None
        matched = match_anchors(self, batch['bb_target'], batch['roi_labels'], box_results_list, img.device)

        class_logits, pred_deltas, seg_logits = self._forward_logits(img)
        batch_class_loss, batch_bbox_loss, monitor = anchor_losses(matched, class_logits, pred_deltas, cf, compute_class_loss, compute_bbox_loss)
        loss = batch_class_loss + batch_bbox_loss
        if self.has_seg_head:
            seg_dice, seg_ce = seg_loss_terms(seg_logits, seg, cf, group=self.seg_loss_group())
            loss = loss + (seg_dice + seg_ce) / 2

        detections = self._detect(class_logits, pred_deltas)
        vals = torch.stack([loss.detach().reshape(()), batch_class_loss.detach().reshape(()), batch_bbox_loss.detach().reshape(())]
                           + ([seg_dice.detach().reshape(()), seg_ce.detach().reshape(())] if self.has_seg_head else []))
        to_host = [detections, vals]
        if self.has_seg_head:
            seg_pred = seg_logits.detach().argmax(1, keepdim=True).to(torch.uint8)        # argmax(softmax) == argmax(logits)
            # "mean pix. pr." of the logger string, reduced on the device (np.mean over the 4 M-voxel label map costs ms of host time per step)
            vals = torch.cat((vals, (seg_pred.sum(dtype=torch.float64) / seg_pred.numel()).to(vals.dtype).reshape(1)))
            to_host = [detections, vals, seg_pred]
        show = kwargs.get('monitor_anchors', True)
        n_host = len(to_host)
        host = self._to_host(to_host + ([t for pair in monitor for t in pair] if show else []))
        results_dict = get_results(cf, img.shape, detections, seg_logits, box_results_list, host=(host[0], host[2] if self.has_seg_head else None))
        if show:
            # positive / sampled-negative anchors for the monitoring plots (retina_unet.py:420-439)
            append_anchor_boxes(self.np_anchors, host[n_host::2], host[n_host + 1::2], img.shape[2:], cf.dim, results_dict['boxes'])
        results_dict['torch_loss'] = loss
        vals = host[1].tolist()
        results_dict['monitor_values'] = {'loss': vals[0], 'class_loss': vals[1]}
        if self.has_seg_head:
            results_dict['logger_string'] = "loss: {0:.2f}, class: {1:.2f}, bbox: {2:.2f}, seg dice: {3:.3f}, seg ce: {4:.3f}, mean pix. pr.: {5:.5f}" \
                .format(vals[0], vals[1], vals[2], vals[3], vals[4], vals[5])
        else:
            results_dict['logger_string'] = "loss: {0:.2f}, class: {1:.2f}, bbox: {2:.2f}".format(vals[0], vals[1], vals[2])
        return results_dict

    def test_forward(self, batch, **kwargs):
        img = self._to_device(batch['data'])
        with torch.no_grad():
            detections, _, _, seg_logits = self.forward(img)
        return get_results(self.cf, img.shape, detections, seg_logits)


batch_dice = mutils.batch_dice
