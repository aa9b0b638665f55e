"""Detection U-Net ("U-Net + heuristics" baseline of the Retina U-Net paper) on libmdt_b200 — the operator surface of the reference's
models/detection_unet.py (`net(cf, logger)` with `forward(x)`, `train_forward(batch)`, `test_forward(batch)`, the same attribute names, state-dict
keys and results_dict format):

  reference (file:line)                                              here
  -----------------------------------------------------------------  ----------------------------------------------------------------------
  FPN(operate_stride1=True) + 1x1 conv_final   detection_unet.py:41-42  same modules/keys, native convs, logits channels-last
  softmax -> host, argmax, get_coords, score loop          :58-85,170-213  one device op (csrc/seg_components.cu), boxes/scores/counts copied
  batch_dice(fp weight) + cross_entropy(weight=wce_weights)      :124-130  fused class-weighted seg loss (csrc/loss_ops.cu), uint8 labels
"""
import numpy as np
import torch

from . import native_ops
from ._detector import Detector
from .backbone import FPN
from .conv import NDConvGenerator, no_split_consumer


def _box_lists(boxes, scores, n_kept, n_fg):
    """device-op outputs (numpy) -> the reference's nested lists: coords[class][element] = int64 array (n, 2*dim) or [] when the element has
    no component of that class; scores[class][element] = list of float32 scores"""
    out_coords, out_scores = [], []
    for c in range(n_fg):
        coords, sc = [], []
        for b in range(boxes.shape[0]):
            n = int(n_kept[b, c])
            coords.append(boxes[b, c, :n].astype(np.int64) if n else [])
            sc.append([np.float32(s) for s in scores[b, c, :n]])
        out_coords.append(coords)
        out_scores.append(sc)
    return out_coords, out_scores


class net(Detector):

    def build(self):
        cf = self.cf
        conv = NDConvGenerator(cf.dim)
        self.fpn = FPN(cf, conv, operate_stride1=True)
        self.conv_final = no_split_consumer(conv(cf.end_filts, cf.num_seg_classes, ks=1, pad=0, norm=cf.norm, relu=None))

    def _logits(self, x):
        return self.conv_final(self.fpn(x)[0])

    def _components(self, seg_logits):
        cf = self.cf
        return native_ops.seg_components(seg_logits.detach(), len(cf.class_dict), cf.n_roi_candidates, median=cf.aggregation_operation == 'median')

    def forward(self, x):
        """x (b, c, y, x, (z)) -> seg_logits (b, n_classes, y, x, (z)); out_box_coords[class][element] = array (n_rois, 2*dim);
        out_max_scores[class][element] = list of n_rois scores"""
        seg_logits = self._logits(x)
        comp = self._components(seg_logits)
        boxes, scores, n_kept = self._to_host([comp['boxes'], comp['scores'], comp['n_kept']])
        coords, sc = _box_lists(boxes, scores, n_kept, len(self.cf.class_dict))
        return seg_logits, coords, sc

    def _det_boxes(self, n_b, coords, scores):
        boxes = [[] for _ in range(n_b)]
        for cix in range(len(self.cf.class_dict)):
            for bix in range(n_b):
                for rix in range(len(scores[cix][bix])):
                    if scores[cix][bix][rix] > self.cf.detection_min_confidence:
                        boxes[bix].append({'box_coords': np.copy(coords[cix][bix][rix]), 'box_score': scores[cix][bix][rix],
                                           'box_pred_class_id': cix + 1, 'box_type': 'det'})
        return boxes

    def seg_loss_terms(self, seg_logits, seg_u8):
        """-> (1 - soft dice with cf.fp_dice_weight, class-weighted cross-entropy), each a differentiable 0-d tensor"""
        cf = self.cf
        w = None
        if 'wce' in cf.seg_loss_mode:
            w = torch.tensor(cf.wce_weights, dtype=torch.float32).to(seg_logits.device, non_blocking=True)
        dice, ce = native_ops.seg_loss(seg_logits, seg_u8, false_positive_weight=float(cf.fp_dice_weight), class_weights=w, group=self.seg_loss_group())
        return 1 - dice, ce

    def train_forward(self, batch, **kwargs):
        """batch {'data', 'seg', 'bb_target', 'roi_labels'} -> results_dict {'boxes', 'seg_preds' (int64), 'torch_loss' [1], 'monitor_values',
        'logger_string'}.  Everything is queued on the device; boxes, scores, counts, the label map and the loss come back after ONE sync."""
        cf = self.cf
        if cf.seg_loss_mode not in ('dice', 'wce', 'dice_wce'):
            raise ValueError("seg_loss_mode must be one of 'dice', 'wce', 'dice_wce'")
        img = self._to_device(batch['data'])
        seg = self._to_device(batch['seg'], dtype=torch.uint8).contiguous()
        n_b = img.shape[0]
        seg_logits = self._logits(img)
        comp = self._components(seg_logits)
        dice_loss, ce_loss = self.seg_loss_terms(seg_logits, seg)
        loss = img.new_zeros(1)
        if cf.seg_loss_mode in ('dice', 'dice_wce'):
            loss = loss + dice_loss
        if cf.seg_loss_mode in ('wce', 'dice_wce'):
            loss = loss + ce_loss
        boxes, scores, n_kept, seg_pred, loss_h = self._to_host([comp['boxes'], comp['scores'], comp['n_kept'], comp['seg_pred'], loss])
        coords, sc = _box_lists(boxes, scores, n_kept, len(cf.class_dict))
        results_dict = {'boxes': self._det_boxes(n_b, coords, sc)}
        for bix in range(n_b):
            for tix in range(len(batch['bb_target'][bix])):
                results_dict['boxes'][bix].append({'box_coords': batch['bb_target'][bix][tix], 'box_label': batch['roi_labels'][bix][tix],
                                                   'box_type': 'gt'})
        results_dict['seg_preds'] = seg_pred[:, np.newaxis].astype(np.int64)
        results_dict['torch_loss'] = loss
        lv = float(loss_h[0])
        results_dict['monitor_values'] = {'loss': lv}
        results_dict['logger_string'] = "loss: {0:.2f}".format(lv)
        return results_dict

    def test_forward(self, batch, **kwargs):
        """batch {'data'} -> results_dict {'boxes', 'seg_preds' (uint8)}"""
        img = self._to_device(batch['data'])
        with torch.no_grad():
            seg_logits = self._logits(img)
            comp = self._components(seg_logits)
            boxes, scores, n_kept, seg_pred = self._to_host([comp['boxes'], comp['scores'], comp['n_kept'], comp['seg_pred']])
        coords, sc = _box_lists(boxes, scores, n_kept, len(self.cf.class_dict))
        return {'boxes': self._det_boxes(img.shape[0], coords, sc), 'seg_preds': seg_pred[:, np.newaxis]}
