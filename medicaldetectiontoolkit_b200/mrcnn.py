"""Mask R-CNN (two-stage detector with mask head) on libmdt_b200 — operator surface of the reference's models/mrcnn.py
(`net(cf, logger)`: `train_forward`, `test_forward`, `forward`, `loss_samples_forward`; module / parameter names identical so state dicts
load key-for-key).

  reference (file:line)                                    here
  -------------------------------------------------------  -----------------------------------------------------------------------
  RPN / Classifier / Mask heads           mrcnn.py:40-169  same modules on tensor-core convs; ConvTranspose3d(k2,s2) = 1x1x1 conv + voxel shuffle
  proposal_layer (sort, NMS 0.7, pad)     :297-369         top-k + csrc/nms.cu with on-device reduction; fixed-shape padding, NO host sync
  pyramid_roi_align                       :373-457         csrc/roi_align.cu (channels-last, 128-bit gathers; fixed-order gather backward)
  detection_target_layer                  :461-613         broadcast IoU, RoIAlign on GT masks, device SHEM
  refine_detections                       :620-714         one batched multi-class NMS launch (groups translated apart), top-k per element
  numpy gt_anchor_matching per element    :894             fp64 device kernels (csrc/anchor_match.cu) on a side stream
"""
import functools

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import model_utils as mutils
from . import native_ops
from ._detector import Detector, anchor_losses, append_anchor_boxes, match_anchors
from .backbone import FPN
from .conv import Conv3d, NDConvGenerator, _Conv3dFn, no_split_consumer
from .native_ops import CropAndResizeFunction as ra3D, CropAndResizeFunction2D as ra2D
from .norm import LeakyReLU
from .retina_unet import compute_bbox_loss as _pos_bbox_loss, compute_class_loss as _shem_class_loss


# ------------------------------------------------------------------------------------------------------------------ heads
class RPN(nn.Module):
    """region proposal head: conv3 -> (1x1 class logits, 1x1 box deltas) per anchor   (mrcnn.py:40-85)"""

    def __init__(self, cf, conv):
        super().__init__()
        self.dim = conv.dim
        self.conv_shared = conv(cf.end_filts, cf.n_rpn_features, ks=3, stride=cf.rpn_anchor_stride, pad=1, relu=cf.relu)
        self.conv_class = no_split_consumer(conv(cf.n_rpn_features, 2 * len(cf.rpn_anchor_ratios), ks=1, stride=1, relu=None))
        self.conv_bbox = no_split_consumer(conv(cf.n_rpn_features, 2 * self.dim * len(cf.rpn_anchor_ratios), ks=1, stride=1, relu=None))

    def forward(self, x):
        x = self.conv_shared(x)
        axes = (0, 2, 3, 1) if self.dim == 2 else (0, 2, 3, 4, 1)
        logits = self.conv_class(x).permute(*axes).contiguous().view(x.size(0), -1, 2)   # channels-last: the permute is a view
        probs = F.softmax(logits, dim=2)
        bbox = self.conv_bbox(x).permute(*axes).contiguous().view(x.size(0), -1, self.dim * 2)
        return [logits, probs, bbox]


class Classifier(nn.Module):
    """RoIAlign -> conv(ks = pool_size) -> 1x1 -> class logits + per-class box deltas   (mrcnn.py:89-126)"""

    def __init__(self, cf, conv):
        super().__init__()
        self.dim = conv.dim
        self.in_channels = cf.end_filts
        self.pool_size = cf.pool_size
        self.pyramid_levels = cf.pyramid_levels
        norm = cf.norm if cf.norm != 'instance_norm' else None
        self.conv1 = conv(cf.end_filts, cf.end_filts * 4, ks=self.pool_size, stride=1, norm=norm, relu=cf.relu)
        self.conv2 = no_split_consumer(conv(cf.end_filts * 4, cf.end_filts * 4, ks=1, stride=1, norm=norm, relu=cf.relu))
        self.linear_class = nn.Linear(cf.end_filts * 4, cf.head_classes)
        self.linear_bbox = nn.Linear(cf.end_filts * 4, cf.head_classes * 2 * self.dim)

    def forward(self, x, rois):
        x = pyramid_roi_align(x, rois, self.pool_size, self.pyramid_levels, self.dim)
        x = self.conv2(self.conv1(x)).reshape(-1, self.in_channels * 4)
        bbox = self.linear_bbox(x)
        return [self.linear_class(x), bbox.view(bbox.size(0), -1, self.dim * 2)]


class _Deconv2x(nn.Module):
    """ConvTranspose{2,3}d(kernel 2, stride 2) with the reference's parameter layout ([Cin, Cout, 2, 2(, 2)] weight, [Cout] bias) computed
    as a 1x1(x1) convolution to 2^dim * Cout channels on the tensor-core conv kernels followed by a voxel shuffle (each input voxel owns a
    disjoint 2^dim output block, so the transposed conv is a plain GEMM)."""

    def __init__(self, c_in, c_out, dim):
        super().__init__()
        self.dim = dim
        self.c_out = c_out
        ref = (nn.ConvTranspose3d if dim == 3 else nn.ConvTranspose2d)(c_in, c_out, kernel_size=2, stride=2)  # same default init / RNG use
        self.weight = nn.Parameter(ref.weight.detach().clone())
        self.bias = nn.Parameter(ref.bias.detach().clone())

    def forward(self, x):
        co, ci = self.c_out, self.weight.shape[0]
        if self.dim == 3:
            w = self.weight.permute(2, 3, 4, 1, 0).reshape(8 * co, ci, 1, 1, 1)
            y = _Conv3dFn.apply(x, w, self.bias.repeat(8), None, (1, 1, 1), (0, 0, 0), False, None, None)
            n, _, d, h, w_ = y.shape
            y = y.view(n, 2, 2, 2, co, d, h, w_).permute(0, 4, 5, 1, 6, 2, 7, 3)
            return y.reshape(n, co, 2 * d, 2 * h, 2 * w_)
        w = self.weight.permute(2, 3, 1, 0).reshape(4 * co, ci, 1, 1, 1)
        y = _Conv3dFn.apply(x.unsqueeze(2), w, self.bias.repeat(4), None, (1, 1, 1), (0, 0, 0), False, None, None).squeeze(2)
        n, _, h, w_ = y.shape
        y = y.view(n, 2, 2, co, h, w_).permute(0, 3, 4, 1, 5, 2)
        return y.reshape(n, co, 2 * h, 2 * w_)


class Mask(nn.Module):
    """RoIAlign -> 4 x conv3 -> deconv x2 -> 1x1 -> sigmoid   (mrcnn.py:130-169)"""

    def __init__(self, cf, conv):
        super().__init__()
        self.pool_size = cf.mask_pool_size
        self.pyramid_levels = cf.pyramid_levels
        self.dim = conv.dim
        self.conv1 = conv(cf.end_filts, cf.end_filts, ks=3, stride=1, pad=1, norm=cf.norm, relu=cf.relu)
        self.conv2 = conv(cf.end_filts, cf.end_filts, ks=3, stride=1, pad=1, norm=cf.norm, relu=cf.relu)
        self.conv3 = conv(cf.end_filts, cf.end_filts, ks=3, stride=1, pad=1, norm=cf.norm, relu=cf.relu)
        self.conv4 = conv(cf.end_filts, cf.end_filts, ks=3, stride=1, pad=1, norm=cf.norm, relu=cf.relu)
        self.deconv = _Deconv2x(cf.end_filts, cf.end_filts, conv.dim)
        self.relu = nn.ReLU(inplace=True) if cf.relu == 'relu' else LeakyReLU(inplace=True)
        self.conv5 = no_split_consumer(conv(cf.end_filts, cf.head_classes, ks=1, stride=1, relu=None))
        self.sigmoid = nn.Sigmoid()

    def forward(self, x, rois):
        x = pyramid_roi_align(x, rois, self.pool_size, self.pyramid_levels, self.dim)
        x = self.conv4(self.conv3(self.conv2(self.conv1(x))))
        x = self.relu(self.deconv(x))
        return self.sigmoid(self.conv5(x))


# ------------------------------------------------------------------------------------------------------------------ losses
def compute_rpn_class_loss(rpn_match, rpn_class_logits, shem_poolsize, max_pos=None, pos_ids=None):
    """CE(positives -> 1) + CE(SHEM negatives -> 0), halved (mrcnn.py:176-213); fixed-shape, sync-free (see retina_unet.compute_class_loss)"""
    return _shem_class_loss(rpn_match, rpn_class_logits, shem_poolsize=shem_poolsize, max_pos=max_pos, pos_ids=pos_ids)


def compute_rpn_bbox_loss(rpn_target_deltas, rpn_pred_deltas, rpn_match, max_pos=None, pos_ids=None):
    """smooth-L1 on positive anchors (mrcnn.py:216-235)"""
    return _pos_bbox_loss(rpn_target_deltas, rpn_pred_deltas, rpn_match, max_pos=max_pos, pos_ids=pos_ids)


def compute_mrcnn_class_loss(target_class_ids, pred_class_logits):
    if target_class_ids.numel() == 0:
        return pred_class_logits.new_zeros(())
    return F.cross_entropy(pred_class_logits, target_class_ids.long())


def compute_mrcnn_bbox_loss(mrcnn_target_deltas, mrcnn_pred_deltas, target_class_ids):
    """smooth-L1 on the class-specific deltas of positive rois (mrcnn.py:251-268); masked mean instead of nonzero()"""
    if target_class_ids.numel() == 0:
        return mrcnn_pred_deltas.new_zeros(())
    pos = (target_class_ids > 0)
    cls = target_class_ids.long().clamp_min(0)
    pred = mrcnn_pred_deltas[torch.arange(cls.shape[0], device=cls.device), cls]
    l = F.smooth_l1_loss(pred, mrcnn_target_deltas.detach(), reduction='none').sum(1)
    return (l * pos).sum() / (pos.sum().clamp_min(1) * pred.shape[1])


def compute_mrcnn_mask_loss(target_masks, pred_masks, target_class_ids):
    """binary CE on the class-specific mask of positive rois (mrcnn.py:271-290)"""
    if target_class_ids.numel() == 0:
        return pred_masks.new_zeros(())
    pos = (target_class_ids > 0)
    cls = target_class_ids.long().clamp_min(0)
    pred = pred_masks[torch.arange(cls.shape[0], device=cls.device), cls]
    bce = F.binary_cross_entropy(pred, target_masks.detach(), reduction='none').flatten(1).mean(1)
    return (bce * pos).sum() / pos.sum().clamp_min(1)


# ------------------------------------------------------------------------------------------------------------------ helper layers
def proposal_layer(rpn_pred_probs, rpn_pred_deltas, proposal_count, anchors, cf):
    """top pre_nms_limit anchors by fg score -> decode, clip -> NMS(rpn_nms_threshold) -> first proposal_count, zero padded, normalised
    (mrcnn.py:297-369).  Everything stays on the device with fixed shapes; returns (boxes [b, P, 2*dim] normalised,
    proposals+score [b, P, 2*dim+1] CUDA tensor — the reference copies this one to numpy for plotting)."""
    dim = cf.dim
    dev = rpn_pred_probs.device
    std_dev = torch.as_tensor(cf.rpn_bbox_std_dev[None], dtype=torch.float32, device=dev)
    norm = torch.as_tensor(np.asarray(cf.scale), dtype=torch.float32, device=dev)
    apply = mutils.apply_box_deltas_2D if dim == 2 else mutils.apply_box_deltas_3D
    clip = mutils.clip_boxes_2D if dim == 2 else mutils.clip_boxes_3D
    out_boxes, out_props = [], []
    for ix in range(rpn_pred_probs.shape[0]):
        k = min(cf.pre_nms_limit, anchors.shape[0])
        scores, order = torch.topk(rpn_pred_probs[ix, :, 1], k, sorted=True)
        boxes = clip(apply(anchors[order], rpn_pred_deltas[ix][order] * std_dev), cf.window)
        keep, num = native_ops.nms_sorted(torch.cat((boxes, scores.unsqueeze(1)), 1).contiguous(), cf.rpn_nms_threshold, dim)
        P = proposal_count
        sel = keep[:P] if k >= P else torch.cat((keep, keep.new_zeros(P - k)))
        valid = (torch.arange(P, device=dev) < num.to(torch.long)).unsqueeze(1)
        sel = sel.clamp(0, k - 1)
        b = torch.where(valid, boxes[sel], boxes.new_zeros(()))
        s = torch.where(valid, scores[sel].unsqueeze(1), scores.new_zeros(()))
        out_props.append(torch.cat((b, s), 1))
        out_boxes.append((b / norm).unsqueeze(0))
    return torch.cat(out_boxes), torch.stack(out_props)


def pyramid_roi_align(feature_maps, rois, pool_size, pyramid_levels, dim):
    """RoIAlign of every roi on the pyramid level chosen from its size: level = round(4 + log2(sqrt(h*w))) clamped (mrcnn.py:373-457).
    rois (n, (y1, x1, y2, x2, (z1, z2), batch_ix)) normalised.  Output [n, C, *pool_size], channels-last."""
    boxes = rois[:, :dim * 2]
    batch_ixs = rois[:, dim * 2]
    h = boxes[:, 2] - boxes[:, 0]
    w = boxes[:, 3] - boxes[:, 1]
    roi_level = (4 + torch.log2(torch.sqrt(h * w))).round().int().clamp(pyramid_levels[0], pyramid_levels[-1])
    if len(pyramid_levels) == 5:
        roi_level[h * w > 0.65] = 5
    # ONE launch over all levels (csrc/roi_align.cu roi_cl4_pyramid): the RoI's CTA reads the geometry of its own level — no boolean-mask
    # gather, no per-level launches, no concat + un-permute (mrcnn.py:405-452), each output row written once
    level_ix = (roi_level - pyramid_levels[0]).clamp(0, len(feature_maps) - 1)
    return native_ops.pyramid_roi_align(list(feature_maps), boxes.detach(), batch_ixs.int(), level_ix, pool_size)


def detection_target_layer(batch_proposals, batch_mrcnn_class_scores, batch_gt_class_ids, batch_gt_boxes, batch_gt_masks, cf):
    """sample positive / SHEM-negative rois per batch element and build their class, box and mask targets (mrcnn.py:461-613).
    batch_gt_masks None: no mask targets (UFRCNN+'s variant, ufrcnn.py:461-587); the fourth result is then None."""
    with_masks = batch_gt_masks is not None
    dev = batch_proposals.device
    dim = cf.dim
    scale = torch.as_tensor(np.asarray(cf.scale), dtype=torch.float32, device=dev)
    pos_ix, neg_ix, deltas_l, masks_l, cls_l = [], [], [], [], []
    positive_count = negative_count = 0
    for b in range(len(batch_gt_class_ids)):
        gt_class_ids = torch.as_tensor(np.asarray(batch_gt_class_ids[b])).int().to(dev)
        sel = batch_proposals[:, -1] == b
        element_ix = torch.nonzero(sel).squeeze(1)
        proposals = batch_proposals[element_ix][:, :-1]
        has_gt = np.any(np.asarray(batch_gt_class_ids[b]) > 0)
        positive_samples = 0
        if has_gt:
            gt_boxes = torch.as_tensor(np.asarray(batch_gt_boxes[b])).float().to(dev) / scale
            if with_masks:
                gt_masks = torch.as_tensor(np.asarray(batch_gt_masks[b])).float().to(dev)  # (n_gt, y, x, (z), c)
            overlaps = mutils.bbox_overlaps(proposals, gt_boxes)
            roi_iou_max = overlaps.max(dim=1)[0]
            positive_idx = torch.nonzero(roi_iou_max >= (0.5 if dim == 2 else 0.3)).squeeze(1)
            negative_idx = torch.nonzero(roi_iou_max < (0.1 if dim == 2 else 0.01)).squeeze(1)
            if positive_idx.numel() > 0:
                want = int(cf.train_rois_per_image * cf.roi_positive_ratio)
                positive_idx = positive_idx[mutils.randperm(positive_idx.numel(), dev)[:want]]
                positive_samples = positive_idx.numel()
                positive_rois = proposals[positive_idx]
                assign = overlaps[positive_idx].max(dim=1)[1]
                deltas = mutils.box_refinement(positive_rois, gt_boxes[assign]) / torch.as_tensor(cf.bbox_std_dev, dtype=torch.float32, device=dev)
                if with_masks:
                    roi_masks = gt_masks[assign][..., 0]
                    box_ids = torch.arange(roi_masks.shape[0], device=dev).int()
                    fn = ra2D(cf.mask_shape[0], cf.mask_shape[1], 0) if dim == 2 else ra3D(cf.mask_shape[0], cf.mask_shape[1], cf.mask_shape[2], 0)
                    masks_l.append(torch.round(fn(roi_masks.unsqueeze(1).contiguous(), positive_rois, box_ids).squeeze(1)))
                pos_ix.append(element_ix[positive_idx])
                deltas_l.append(deltas)
                cls_l.append(gt_class_ids[assign])
                positive_count += positive_samples
        else:
            negative_idx = torch.arange(proposals.shape[0], device=dev)
        if negative_idx.numel() > 0:
            r = 1.0 / cf.roi_positive_ratio
            b_neg = max(int(r * positive_samples - positive_samples), 1)
            picked = mutils.shem(batch_mrcnn_class_scores[element_ix[negative_idx]], b_neg, cf.shem_poolsize)
            neg_ix.append(element_ix[negative_idx[picked]])
            negative_count += picked.numel()
    mask_shape = tuple(cf.mask_shape)
    parts_ix = pos_ix + neg_ix
    if not parts_ix:
        return (torch.zeros(0, dtype=torch.long, device=dev), torch.zeros(0, dtype=torch.int32, device=dev),
                torch.zeros((0, dim * 2), device=dev), torch.zeros((0,) + mask_shape, device=dev) if with_masks else None)
    sample_indices = torch.cat(parts_ix)
    target_class_ids = torch.cat(cls_l + [torch.zeros(negative_count, dtype=torch.int32, device=dev)])
    target_deltas = torch.cat(deltas_l + [torch.zeros((negative_count, dim * 2), device=dev)])
    target_masks = torch.cat(masks_l + [torch.zeros((negative_count,) + mask_shape, device=dev)]) if with_masks else None
    return sample_indices, target_class_ids, target_deltas, target_masks


def refine_detections(rois, probs, deltas, batch_ixs, cf):
    """per foreground class: decode the class-specific deltas, clip, round, drop scores < model_min_confidence, NMS per (element, class),
    top model_max_instances_per_batch_element per element (mrcnn.py:620-714) — as one batched NMS launch, fixed shapes until the final gather."""
    dim = cf.dim
    dev = rois.device
    n = rois.shape[0]
    fg = cf.head_classes - 1
    class_ids = torch.arange(1, fg + 1, device=dev).repeat_interleave(n)
    idx = torch.arange(n, device=dev).repeat(fg)
    scores_all = probs[idx, class_ids]
    b_all = batch_ixs[idx]
    std_dev = torch.as_tensor(np.reshape(cf.rpn_bbox_std_dev, [1, dim * 2]), dtype=torch.float32, device=dev)
    scale = torch.as_tensor(np.asarray(cf.scale), dtype=torch.float32, device=dev)
    apply = mutils.apply_box_deltas_2D if dim == 2 else mutils.apply_box_deltas_3D
    refined = torch.round(mutils.clip_to_window(cf.window, apply(rois[idx], deltas[idx, class_ids] * std_dev) * scale))
    # sort all candidates by score once; low-confidence ones sink to the end with score -1 and are dropped by the validity mask
    conf = scores_all >= cf.model_min_confidence
    key = torch.where(conf, scores_all, scores_all.new_full((), -1.0))
    s_sorted, order = key.sort(descending=True)
    r_sorted, c_sorted, b_sorted = refined[order], class_ids[order], b_all[order].long()
    band = float(max(cf.window[2], cf.window[3]) + 2)
    offs = (b_sorted * (fg + 1) + c_sorted).to(r_sorted.dtype) * band + torch.where(s_sorted < 0, band * 1e3, 0.0)
    shifted = r_sorted.clone()
    shifted[:, 0] += offs
    shifted[:, 2] += offs
    keep_pad, num = native_ops.nms_sorted(torch.cat((shifted, s_sorted.unsqueeze(1)), 1).contiguous(), cf.detection_nms_threshold, dim)
    m = s_sorted.shape[0]
    kept = torch.zeros(m, dtype=torch.bool, device=dev)
    valid = torch.arange(m, device=dev) < num.to(torch.long)
    kept[keep_pad.clamp(0, m - 1)[valid]] = True
    kept &= s_sorted >= 0
    n_b = int(batch_ixs.max().item()) + 1 if batch_ixs.numel() else 1
    onehot = (b_sorted.unsqueeze(0) == torch.arange(n_b, device=dev).unsqueeze(1)) & kept.unsqueeze(0)   # [n_b, m]: scan along the contiguous dim
    within = (torch.cumsum(onehot.to(torch.int32), 1) * onehot).sum(0)
    final = kept & (within <= cf.model_max_instances_per_batch_element)
    sel = torch.nonzero(final).squeeze(1)
    if sel.numel() == 0:   # the reference falls back to candidate 0 (mrcnn.py:706)
        return torch.cat((refined[:1], b_all[:1].unsqueeze(1).float(), class_ids[:1].unsqueeze(1).float(), scores_all[:1].unsqueeze(1)), 1)
    return torch.cat((r_sorted[sel], b_sorted[sel].unsqueeze(1).float(), c_sorted[sel].unsqueeze(1).float(), s_sorted[sel].unsqueeze(1)), 1)


def unmold_seg(img_shape, detections, detection_masks):
    """seg_preds on the device: uint8 [b, 1, *spatial], the union of the detections' masks resized to their boxes (csrc/unmold.cu; the reference
    resizes each mask with scipy on the host, utils/model_utils.py:147-183)"""
    return native_ops.unmold_masks(detections, detection_masks, img_shape).unsqueeze(1)


def get_results(cf, img_shape, detections, detection_masks, box_results_list=None, return_masks=True, host=None):
    """results_dict {'boxes', 'seg_preds'} (mrcnn.py:717-799).
    host: optional (detections, seg_preds) numpy arrays already copied to the host (train_forward and test_forward batch their device->host
    copies; seg_preds is unmold_seg's result, or None without return_masks)"""
    dim = cf.dim
    if host is None:
        seg = unmold_seg(img_shape, detections, detection_masks) if return_masks else None
        host = (detections.detach().cpu().numpy(), None if seg is None else seg.cpu().numpy())
    det = host[0]
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
        ok = vol > 0
        for bx, s, c in zip(boxes[ok], scores[ok], class_ids[ok]):
            box_results_list[ix].append({'box_coords': bx, 'box_score': s, 'box_type': 'det', 'box_pred_class_id': c})
    seg_preds = host[1] if host[1] is not None else np.zeros((img_shape[0], 1) + tuple(img_shape[2:]), dtype=np.uint8)
    return {'boxes': box_results_list, 'seg_preds': seg_preds}


def first_stage(net, fmaps, is_training):
    """RPN on every pyramid level, proposals and the gradient-free classifier pass over all proposals in roi_chunk_size chunks (mrcnn.py:
    987-1036).  Sets net.mrcnn_feature_maps, net.rpn_rois_batch_info and net.batch_mrcnn_class_scores for loss_samples_forward.
    -> (rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, arguments of refine_detections without cf)"""
    cf = net.cf
    net.mrcnn_feature_maps = fmaps
    outs = list(zip(*[net.rpn(p) for p in fmaps]))
    rpn_pred_logits, rpn_pred_probs, rpn_pred_deltas = [torch.cat(list(o), dim=1) for o in outs]
    proposal_count = cf.post_nms_rois_training if is_training else cf.post_nms_rois_inference
    with torch.no_grad():
        batch_rpn_rois, batch_proposal_boxes = proposal_layer(rpn_pred_probs.detach(), rpn_pred_deltas.detach(), proposal_count, net.anchors, cf)
        b, P = batch_rpn_rois.shape[0], batch_rpn_rois.shape[1]
        batch_ixs = torch.arange(b, device=batch_rpn_rois.device).repeat_interleave(P).float()
        rpn_rois = batch_rpn_rois.view(-1, batch_rpn_rois.shape[2])
        net.rpn_rois_batch_info = torch.cat((rpn_rois, batch_ixs.unsqueeze(1)), dim=1)
        logits_l, bbox_l = [], []
        for chunk in net.rpn_rois_batch_info.split(cf.roi_chunk_size):
            cl, bb = net.classifier(fmaps, chunk)
            logits_l.append(cl)
            bbox_l.append(bb)
        net.batch_mrcnn_class_scores = F.softmax(torch.cat(logits_l, 0), dim=1)
    return rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, (rpn_rois, net.batch_mrcnn_class_scores, torch.cat(bbox_l, 0), batch_ixs)


def append_proposal_boxes(host_props, host_rois, host_t_cls, cf, box_results_list):
    """the top n_plot_rpn_props proposals of each element and the second stage's positive / negative samples for the monitoring plots
    (mrcnn.py:904-916), from host copies of the proposals, the window-clipped sampled rois and their target class ids"""
    for b, props in enumerate(host_props):
        for r in props[props[:, -1].argsort()][::-1][:cf.n_plot_rpn_props, :-1]:
            box_results_list[b].append({'box_coords': r, 'box_type': 'prop'})
    for ix, r in enumerate(host_rois):
        box_results_list[int(r[-1])].append({'box_coords': r[:-1] * cf.scale, 'box_type': 'pos_class' if host_t_cls[ix] > 0 else 'neg_class'})


# ------------------------------------------------------------------------------------------------------------------ net
class net(Detector):

    def build(self):
        cf = self.cf
        self._check_patch_size(check_z=True)
        conv = NDConvGenerator(cf.dim)
        self._register_anchors()
        self.fpn = FPN(cf, conv, operate_stride1=False)
        self.rpn = RPN(cf, conv)
        self.classifier = Classifier(cf, conv)
        self.mask = Mask(cf, conv)

    def forward(self, img, is_training=True):
        """-> [rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, detections, detection_masks] (mrcnn.py:987-1049)"""
        cf = self.cf
        fpn_outs = self.fpn(img)
        rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, refine_args = first_stage(self, [fpn_outs[i] for i in cf.pyramid_levels], is_training)
        with torch.no_grad():
            detections = refine_detections(*refine_args, cf)
            sp = list(img.shape[2:])
            scale = torch.as_tensor([sp[0], sp[1], sp[0], sp[1]] + ([sp[2], sp[2]] if cf.dim == 3 else []) + [1], dtype=torch.float32, device=img.device)
            detection_masks = self.mask(self.mrcnn_feature_maps, detections[:, :cf.dim * 2 + 1] / scale)
        return [rpn_pred_logits, rpn_pred_deltas, batch_proposal_boxes, detections, detection_masks]

    def loss_samples_forward(self, batch_gt_class_ids, batch_gt_boxes, batch_gt_masks):
        """second pass through the second stage on the sampled rois, with gradients (mrcnn.py:1052-1083)"""
        with torch.no_grad():
            sample_ix, t_cls, t_deltas, t_mask = detection_target_layer(self.rpn_rois_batch_info, self.batch_mrcnn_class_scores, batch_gt_class_ids,
                                                                        batch_gt_boxes, batch_gt_masks, self.cf)
        sample_proposals = self.rpn_rois_batch_info[sample_ix]
        if sample_proposals.shape[0] > 0:
            logits, boxes = self.classifier(self.mrcnn_feature_maps, sample_proposals)
            mask = self.mask(self.mrcnn_feature_maps, sample_proposals)
        else:
            dev = sample_proposals.device
            logits, boxes, mask = torch.zeros(0, device=dev), torch.zeros(0, device=dev), torch.zeros(0, device=dev)
        return [logits, boxes, mask, t_cls, t_deltas, t_mask, sample_proposals]

    def train_forward(self, batch, is_validation=False, **kwargs):
        """batch {'data', 'seg', 'bb_target', 'roi_labels', 'roi_masks'} -> results_dict {'boxes', 'seg_preds', 'torch_loss', 'monitor_values',
        'logger_string'} (mrcnn.py:853-966).  The RPN matching (and its host waits) runs first on a side stream; the network and every loss
        are then queued; the detections, loss values, sample classes and monitoring boxes come back in one batched device->host copy."""
        cf = self.cf
        gt_class_ids, gt_boxes = batch['roi_labels'], batch['bb_target']
        axes = (0, 2, 3, 1) if cf.dim == 2 else (0, 2, 3, 4, 1)
        gt_masks = [np.transpose(batch['roi_masks'][ii], axes=axes) for ii in range(len(batch['roi_masks']))]
        img = self._to_device(batch['data'])
        box_results_list = [[] for _ in range(img.shape[0])]
        matched = match_anchors(self, gt_boxes, gt_class_ids, box_results_list, img.device, class_agnostic=True)
        rpn_class_logits, rpn_pred_deltas, proposal_boxes, detections, detection_masks = self.forward(img)
        logits, pred_deltas, pred_mask, t_cls, t_deltas, t_mask, sample_proposals = self.loss_samples_forward(gt_class_ids, gt_boxes, gt_masks)
        rpn_class_loss, rpn_bbox_loss, monitor = anchor_losses(matched, rpn_class_logits, rpn_pred_deltas, cf,
                                                               functools.partial(compute_rpn_class_loss, shem_poolsize=cf.shem_poolsize),
                                                               compute_rpn_bbox_loss)
        mrcnn_class_loss = compute_mrcnn_class_loss(t_cls, logits)
        mrcnn_bbox_loss = compute_mrcnn_bbox_loss(t_deltas, pred_deltas, t_cls)
        mrcnn_mask_loss = compute_mrcnn_mask_loss(t_mask, pred_mask, t_cls) if not cf.frcnn_mode else img.new_zeros(())
        loss = rpn_class_loss + rpn_bbox_loss + mrcnn_class_loss + mrcnn_bbox_loss + mrcnn_mask_loss

        vals = torch.stack([v.detach().reshape(()) for v in (loss, rpn_class_loss, rpn_bbox_loss, mrcnn_class_loss, mrcnn_bbox_loss, mrcnn_mask_loss)])
        dcount = torch.stack([(t_cls == c).sum() for c in range(1, cf.head_classes)])
        show = kwargs.get('monitor_anchors', True)
        return_masks = cf.return_masks_in_val if is_validation else False
        to_host = [detections, vals, dcount] + ([unmold_seg(img.shape, detections, detection_masks)] if return_masks else [])
        n_host = len(to_host)
        if show:
            to_host += [t_cls, proposal_boxes, mutils.clip_to_window(cf.window, sample_proposals.clone())] + [t for pair in monitor for t in pair]
        host = self._to_host(to_host)
        if show:
            # positive / sampled-negative anchors of the RPN loss, top proposals and the second-stage samples (mrcnn.py:896-916)
            append_anchor_boxes(self.np_anchors, host[n_host + 3::2], host[n_host + 4::2], img.shape[2:], cf.dim, box_results_list)
            append_proposal_boxes(host[n_host + 1], host[n_host + 2], host[n_host], cf, box_results_list)
        results_dict = get_results(cf, img.shape, detections, detection_masks, box_results_list, return_masks=return_masks,
                                   host=(host[0], host[3] if return_masks else None))
        results_dict['torch_loss'] = loss
        vals = host[1].tolist()
        results_dict['monitor_values'] = {'loss': vals[0], 'class_loss': vals[3]}
        results_dict['logger_string'] = "loss: {0:.2f}, rpn_class: {1:.2f}, rpn_bbox: {2:.2f}, mrcnn_class: {3:.2f}, mrcnn_bbox: {4:.2f}, " \
                                        "mrcnn_mask: {5:.2f}, dcount {6}".format(*vals, host[2].tolist())
        return results_dict

    def test_forward(self, batch, return_masks=True):
        img = self._to_device(batch['data'])
        with torch.no_grad():
            _, _, _, detections, detection_masks = self.forward(img, is_training=False)
            to_host = [detections] + ([unmold_seg(img.shape, detections, detection_masks)] if return_masks else [])
        host = self._to_host(to_host)
        return get_results(self.cf, img.shape, detections, detection_masks, return_masks=return_masks,
                           host=(host[0], host[1] if return_masks else None))
