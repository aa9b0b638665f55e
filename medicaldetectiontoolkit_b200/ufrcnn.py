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
import functools

import torch

from . import model_utils as mutils
from . import mrcnn as _mrcnn
from . import retina_unet as _retina
from ._detector import Detector, anchor_losses, append_anchor_boxes, match_anchors, seg_loss_terms
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


class net(Detector):

    def build(self):
        """module creation order fpn, rpn, classifier, mask, final_conv: the reference's, so a seeded build draws the same parameters"""
        cf = self.cf
        self._check_patch_size()
        conv = NDConvGenerator(cf.dim)
        self._register_anchors()
        self.fpn = FPN(cf, conv, operate_stride1=True)
        self.rpn = RPN(cf, conv)
        self.classifier = Classifier(cf, conv)
        self.mask = Mask(cf, conv)            # in the state dict, never called (ufrcnn.py:798)
        self.final_conv = no_split_consumer(conv(cf.end_filts, cf.num_seg_classes, ks=1, pad=0, norm=cf.norm, relu=None))

    def _first_stage(self, img, is_training):
        """backbone, seg head and the Mask R-CNN first stage on P2..P5 (mrcnn.first_stage) -> (rpn logits, rpn deltas, proposal boxes,
        seg logits, arguments of refine_detections)"""
        fpn_outs = self.fpn(img)
        seg_logits = self.final_conv(fpn_outs[0])
        rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, refine_args = _mrcnn.first_stage(
            self, [fpn_outs[i + 1] for i in self.cf.pyramid_levels], is_training)
        return rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, seg_logits, refine_args

    def _detect(self, refine_args):
        with torch.no_grad():
            return refine_detections(*refine_args, self.cf)

    def forward(self, img, is_training=True):
        """-> [rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, detections, seg_logits] (ufrcnn.py:934-988)"""
        rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, seg_logits, refine_args = self._first_stage(img, is_training)
        return [rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, self._detect(refine_args), seg_logits]

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
        seg = self._seg_to_device(batch['seg'], _retina.FUSED_LOSSES)
        box_results_list = [[] for _ in range(img.shape[0])]
        matched = match_anchors(self, gt_boxes, gt_class_ids, box_results_list, img.device, class_agnostic=True)

        rpn_class_logits, rpn_pred_deltas, proposal_boxes, seg_logits, refine_args = self._first_stage(img, True)
        logits, pred_deltas, t_cls, t_deltas, sample_proposals = self.loss_samples_forward(gt_class_ids, gt_boxes)
        rpn_class_loss, rpn_bbox_loss, monitor = anchor_losses(matched, rpn_class_logits, rpn_pred_deltas, cf,
                                                               functools.partial(compute_rpn_class_loss, shem_poolsize=cf.shem_poolsize),
                                                               compute_rpn_bbox_loss)
        mrcnn_class_loss = compute_mrcnn_class_loss(t_cls, logits)
        mrcnn_bbox_loss = compute_mrcnn_bbox_loss(t_deltas, pred_deltas, t_cls)
        seg_dice, seg_ce = seg_loss_terms(seg_logits, seg, cf, group=self.seg_loss_group())
        loss = rpn_class_loss + rpn_bbox_loss + mrcnn_class_loss + mrcnn_bbox_loss + (seg_dice + seg_ce) / 2
        detections = self._detect(refine_args)

        vals = torch.stack([v.detach().reshape(()).float() for v in (loss, rpn_class_loss, rpn_bbox_loss, mrcnn_class_loss, mrcnn_bbox_loss, seg_dice)])
        seg_pred = seg_logits.detach().argmax(1, keepdim=True).to(torch.uint8)              # argmax(softmax) == argmax(logits)
        show = kwargs.get('monitor_anchors', True)
        to_host = [detections, vals, seg_pred, t_cls]
        if show:
            to_host += [proposal_boxes, mutils.clip_to_window(cf.window, sample_proposals.clone())] + [t for pair in monitor for t in pair]
        host = self._to_host(to_host)
        if show:
            # positive / sampled-negative anchors of the RPN loss, top proposals and the second-stage samples (ufrcnn.py:847-880)
            append_anchor_boxes(self.np_anchors, host[6::2], host[7::2], img.shape[2:], cf.dim, box_results_list)
            _mrcnn.append_proposal_boxes(host[4], host[5], host[3], cf, box_results_list)

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
