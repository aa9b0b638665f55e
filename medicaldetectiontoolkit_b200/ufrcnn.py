"""UFRCNN+ (Faster R-CNN + the Retina U-Net full-resolution segmentation head) on libmdt_b200 — operator surface of the reference's
models/ufrcnn.py (`net(cf, logger)`: `forward`, `train_forward`, `test_forward`, `loss_samples_forward`; module / parameter names identical so
state dicts load key-for-key).

  reference (file:line)                                      here
  ---------------------------------------------------------  ---------------------------------------------------------------------------
  RPN / Classifier / Mask, proposal_layer, pyramid_roi_align,  the Mask R-CNN port (mrcnn.py here); the Mask head is built as in the reference
  refine_detections, RPN and second-stage losses               but never called, so its parameters never get a gradient
  FPN(operate_stride1=True) + 1x1 final_conv on P0  :795-799  same modules, native convs; RPN / RoIAlign on P2..P5 (fpn_outs[1:])
  detection_target_layer without GT masks           :461-587  mrcnn.detection_target_layer with batch_gt_masks=None
  1 - batch_dice(softmax, one-hot) + cross_entropy  :896-897  fused seg loss (csrc/loss_ops.cu) on uint8 labels, no one-hot / probabilities
  get_results                                       :691-754  retina_unet.get_results (zero-volume + confidence filter, argmax seg_preds)
  numpy gt_anchor_matching per element              :845      fp64 device kernels on a side stream, before the network is queued
"""
import contextlib

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import model_utils as mutils
from . import mrcnn as _mrcnn
from . import native_ops
from . import retina_unet as _retina
from .backbone import FPN
from .conv import NDConvGenerator, no_split_consumer
from .mrcnn import (RPN, Classifier, Mask, compute_mrcnn_bbox_loss, compute_mrcnn_class_loss, compute_rpn_bbox_loss,  # noqa: F401
                    compute_rpn_class_loss, proposal_layer, pyramid_roi_align, refine_detections)


def detection_target_layer(batch_proposals, batch_mrcnn_class_scores, batch_gt_class_ids, batch_gt_boxes, cf):
    """sample positive / SHEM-negative rois per batch element and build their class and box targets (ufrcnn.py:461-587)
    -> (sample_indices, target_class_ids, target_deltas)"""
    return _mrcnn.detection_target_layer(batch_proposals, batch_mrcnn_class_scores, batch_gt_class_ids, batch_gt_boxes, None, cf)[:3]


# results_dict {'boxes', 'seg_preds'} of ufrcnn.py:691-754: the same filters and label map as the Retina U-Net's
get_results = _retina.get_results


class net(nn.Module):

    def __init__(self, cf, logger=None):
        super().__init__()
        self.cf = cf
        self.logger = logger
        self.build()
        if getattr(cf, 'weight_init', None) is not None:
            if logger is not None:
                logger.info("using pytorch weight init of type {}".format(cf.weight_init))
            mutils.initialize_weights(self)                       # ufrcnn.py:771-775
        elif logger is not None:
            logger.info("using default pytorch weight init")

    def build(self):
        """module creation order fpn, rpn, classifier, mask, final_conv: the reference's, so a seeded build draws the same parameters"""
        cf = self.cf
        h, w = cf.patch_size[:2]
        if h / 2 ** 5 != int(h / 2 ** 5) or w / 2 ** 5 != int(w / 2 ** 5):
            raise Exception("Image size must be dividable by 2 at least 5 times to avoid fractions when downscaling and upscaling.")
        conv = NDConvGenerator(cf.dim)
        self.np_anchors = mutils.generate_pyramid_anchors(self.logger, cf)
        self.register_buffer("anchors", torch.from_numpy(self.np_anchors).float(), persistent=False)
        self.register_buffer("anchors_f64", torch.from_numpy(self.np_anchors).double(), persistent=False)
        self.fpn = FPN(cf, conv, operate_stride1=True)
        self.rpn = RPN(cf, conv)
        self.classifier = Classifier(cf, conv)
        self.mask = Mask(cf, conv)            # in the state dict, never called (ufrcnn.py:798)
        self.final_conv = no_split_consumer(conv(cf.end_filts, cf.num_seg_classes, ks=1, pad=0, norm=cf.norm, relu=None))

    _to_device = _mrcnn.net._to_device
    _to_host = _retina.net._to_host

    def _first_stage(self, img, is_training):
        """backbone, seg head, RPN, proposals and the gradient-free second-stage pass over every proposal; sets rpn_rois_batch_info,
        batch_mrcnn_class_scores and mrcnn_feature_maps for loss_samples_forward.  -> (rpn logits, rpn deltas, proposal boxes, seg logits,
        arguments of refine_detections)"""
        cf = self.cf
        fpn_outs = self.fpn(img)
        seg_logits = self.final_conv(fpn_outs[0])
        fmaps = [fpn_outs[i + 1] for i in cf.pyramid_levels]
        self.mrcnn_feature_maps = fmaps
        outs = list(zip(*[self.rpn(p) for p in fmaps]))
        rpn_pred_logits, rpn_pred_probs, rpn_pred_deltas = [torch.cat(list(o), dim=1) for o in outs]
        proposal_count = cf.post_nms_rois_training if is_training else cf.post_nms_rois_inference
        with torch.no_grad():
            batch_rpn_rois, batch_proposal_boxes = proposal_layer(rpn_pred_probs.detach(), rpn_pred_deltas.detach(), proposal_count, self.anchors, cf)
            b, P = batch_rpn_rois.shape[0], batch_rpn_rois.shape[1]
            batch_ixs = torch.arange(b, device=img.device).repeat_interleave(P).float()
            rpn_rois = batch_rpn_rois.view(-1, batch_rpn_rois.shape[2])
            self.rpn_rois_batch_info = torch.cat((rpn_rois, batch_ixs.unsqueeze(1)), dim=1)
            logits_l, bbox_l = [], []
            for chunk in self.rpn_rois_batch_info.split(cf.roi_chunk_size):
                cl, bb = self.classifier(fmaps, chunk)
                logits_l.append(cl)
                bbox_l.append(bb)
            self.batch_mrcnn_class_scores = F.softmax(torch.cat(logits_l, 0), dim=1)
        return rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, seg_logits, (rpn_rois, torch.cat(bbox_l, 0), batch_ixs)

    def _detect(self, rpn_rois, mrcnn_bbox, batch_ixs):
        with torch.no_grad():
            return refine_detections(rpn_rois, self.batch_mrcnn_class_scores, mrcnn_bbox, batch_ixs, self.cf)

    def forward(self, img, is_training=True):
        """-> [rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, detections, seg_logits] (ufrcnn.py:934-988)"""
        rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, seg_logits, refine_args = self._first_stage(img, is_training)
        return [rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, self._detect(*refine_args), seg_logits]

    def loss_samples_forward(self, batch_gt_class_ids, batch_gt_boxes):
        """second pass through the classifier on the sampled rois, with gradients (ufrcnn.py:991-1019)
        -> [logits, boxes, target_class_ids, target_deltas, sample_proposals]"""
        with torch.no_grad():
            sample_ix, t_cls, t_deltas = detection_target_layer(self.rpn_rois_batch_info, self.batch_mrcnn_class_scores, batch_gt_class_ids,
                                                                batch_gt_boxes, self.cf)
        sample_proposals = self.rpn_rois_batch_info[sample_ix]
        if sample_proposals.shape[0] > 0:
            logits, boxes = self.classifier(self.mrcnn_feature_maps, sample_proposals)
        else:
            dev = sample_proposals.device
            logits, boxes = torch.zeros(0, device=dev), torch.zeros(0, device=dev)
        return [logits, boxes, t_cls, t_deltas, sample_proposals]

    def train_forward(self, batch, is_validation=False, **kwargs):
        """batch {'data', 'seg', 'bb_target', 'roi_labels'} -> results_dict {'boxes', 'seg_preds', 'torch_loss', 'monitor_values',
        'logger_string'} (ufrcnn.py:802-913).  The anchor matching (and its host waits) runs first on a side stream; the network and every
        loss are then queued; the detections, loss values, label map and monitoring boxes come back in one batched device->host copy."""
        cf = self.cf
        gt_class_ids, gt_boxes = batch['roi_labels'], batch['bb_target']
        img = self._to_device(batch['data'])
        n_b = img.shape[0]
        dev = img.device
        fused_seg = _retina.FUSED_LOSSES and img.is_cuda and cf.num_seg_classes <= 8
        seg = self._to_device(batch['seg'], dtype=torch.uint8 if fused_seg else torch.long)   # (b, 1, y, x, (z)) class ids
        box_results_list = [[] for _ in range(n_b)]

        main_stream = torch.cuda.current_stream(dev) if img.is_cuda else None
        match_stream = _retina._side_stream(dev) if main_stream is not None else None
        matched = []
        with (torch.cuda.stream(match_stream) if main_stream is not None else contextlib.nullcontext()):
            for b in range(n_b):
                if len(gt_boxes[b]) > 0:
                    for ix in range(len(gt_boxes[b])):
                        box_results_list[b].append({'box_coords': gt_boxes[b][ix], 'box_label': gt_class_ids[b][ix], 'box_type': 'gt'})
                    matched.append(mutils.gt_anchor_matching_device(cf, self.anchors_f64, gt_boxes[b], return_pos=True))   # class-agnostic
                else:
                    matched.append((torch.full((self.anchors.shape[0],), -1, dtype=torch.int32, device=dev),
                                    torch.zeros((cf.rpn_train_anchors_per_image, 2 * cf.dim), dtype=torch.float64, device=dev),
                                    torch.zeros(0, dtype=torch.long, device=dev)))
        if main_stream is not None:
            main_stream.wait_stream(match_stream)              # the losses (main stream) consume the matching's tensors
            for tup in matched:
                for t in tup:
                    t.record_stream(main_stream)

        rpn_class_logits, rpn_pred_deltas, proposal_boxes, seg_logits, refine_args = self._first_stage(img, True)
        logits, pred_deltas, t_cls, t_deltas, sample_proposals = self.loss_samples_forward(gt_class_ids, gt_boxes)

        max_pos = max(1, cf.rpn_train_anchors_per_image // 2)
        rpn_class_loss = img.new_zeros(1)
        rpn_bbox_loss = img.new_zeros(1)
        monitor = []
        for b, (rpn_match, rpn_target_deltas, pos_ids) in enumerate(matched):
            cl, neg_ix = compute_rpn_class_loss(rpn_match, rpn_class_logits[b], cf.shem_poolsize, max_pos=max_pos, pos_ids=pos_ids)
            monitor += [rpn_match, neg_ix]
            rpn_class_loss = rpn_class_loss + cl / n_b
            rpn_bbox_loss = rpn_bbox_loss + compute_rpn_bbox_loss(rpn_target_deltas, rpn_pred_deltas[b], rpn_match, max_pos=max_pos, pos_ids=pos_ids) / n_b
        mrcnn_class_loss = compute_mrcnn_class_loss(t_cls, logits)
        mrcnn_bbox_loss = compute_mrcnn_bbox_loss(t_deltas, pred_deltas, t_cls)
        if fused_seg:
            # one pass over the logits and the uint8 labels each way (csrc/loss_ops.cu), as in the Retina U-Net
            dice_score, seg_ce = native_ops.seg_loss(seg_logits, seg.contiguous())
            seg_dice = 1 - dice_score
        else:
            seg_ohe = F.one_hot(seg[:, 0], cf.num_seg_classes).movedim(-1, 1).float()
            seg_dice = 1 - mutils.batch_dice(F.softmax(seg_logits, dim=1), seg_ohe)
            seg_ce = F.cross_entropy(seg_logits, seg[:, 0])
        loss = rpn_class_loss + rpn_bbox_loss + mrcnn_class_loss + mrcnn_bbox_loss + (seg_dice + seg_ce) / 2
        detections = self._detect(*refine_args)

        vals = torch.stack([v.detach().reshape(()).float() for v in (loss, rpn_class_loss, rpn_bbox_loss, mrcnn_class_loss, mrcnn_bbox_loss, seg_dice)])
        seg_pred = seg_logits.detach().argmax(1, keepdim=True).to(torch.uint8)              # argmax(softmax) == argmax(logits)
        show = kwargs.get('monitor_anchors', True)
        to_host = [detections, vals, seg_pred, t_cls]
        if show:
            to_host += [proposal_boxes, mutils.clip_to_window(cf.window, sample_proposals.clone())] + monitor
        host = self._to_host(to_host)

        if show:
            # positive / sampled-negative anchors of the RPN loss, top proposals and the second-stage samples (ufrcnn.py:847-880)
            sp = img.shape[2:]
            hi = np.array([sp[0], sp[1], sp[0], sp[1]] + ([sp[2], sp[2]] if cf.dim == 3 else []))
            props, rois = host[4], host[5]
            for b in range(n_b):
                m, nix = host[6 + 2 * b], host[7 + 2 * b]
                for p_ in np.clip(self.np_anchors[m == 1], 0, hi):
                    box_results_list[b].append({'box_coords': p_, 'box_type': 'pos_anchor'})
                neg_all = np.where(m == -1)[0]
                if neg_all.size:
                    for n_ in np.clip(self.np_anchors[neg_all[nix[nix >= 0]]], 0, hi):
                        box_results_list[b].append({'box_coords': n_, 'box_type': 'neg_anchor'})
                for r in props[b][props[b][:, -1].argsort()][::-1][:cf.n_plot_rpn_props, :-1]:
                    box_results_list[b].append({'box_coords': r, 'box_type': 'prop'})
            for ix, r in enumerate(rois):
                box_results_list[int(r[-1])].append({'box_coords': r[:-1] * cf.scale, 'box_type': 'pos_class' if host[3][ix] > 0 else 'neg_class'})

        results_dict = get_results(cf, img.shape, detections, seg_logits, box_results_list, host=(host[0], host[2]))
        results_dict['torch_loss'] = loss
        v = host[1].tolist()
        dcount = [int((host[3] == c).sum()) for c in range(1, cf.head_classes)]
        results_dict['monitor_values'] = {'loss': v[0], 'class_loss': v[3]}
        results_dict['logger_string'] = "loss: {0:.2f}, rpn_class: {1:.2f}, rpn_bbox: {2:.2f}, mrcnn_class: {3:.2f}, mrcnn_bbox: {4:.2f}, " \
                                        "dice_loss: {5:.2f}, dcount {6}".format(*v, dcount)
        return results_dict

    def test_forward(self, batch, return_masks=True):
        """batch {'data'} -> results_dict {'boxes', 'seg_preds'} (ufrcnn.py:916-931).  return_masks is ignored, and the proposal count is
        post_nms_rois_training, as in the reference (its forward runs with the default is_training=True)."""
        img = self._to_device(batch['data'])
        with torch.no_grad():
            _, _, _, detections, seg_logits = self.forward(img)
            seg_pred = seg_logits.argmax(1, keepdim=True).to(torch.uint8)
            host = self._to_host([detections, seg_pred])
        return get_results(self.cf, img.shape, detections, seg_logits, host=host)
