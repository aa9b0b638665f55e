"""Train-step plumbing shared by the detection models (retina_unet / retina_net, mrcnn, ufrcnn, detection_unet): construction and weight
init, host<->device transfers, GT<->anchor matching on a side stream, the per-element anchor losses, the seg loss of the Retina U-Net and
UFRCNN+, and the anchor boxes of the monitoring plots.  The model modules keep their own heads, losses and results; the loss functions are
passed in by the caller, so a model module's globals stay the names that are called."""
import contextlib

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import model_utils as mutils
from . import native_ops

_SIDE_STREAMS = {}
_PINNED = {}      # pinned device->host staging buffers of train_forward, keyed by (net, slot, shape, dtype)


def _side_stream(dev):
    """one side stream per device for the GT<->anchor matching (kept out of the module so that nets stay picklable / deep-copyable)"""
    key = (dev.type, dev.index)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=dev)
    return _SIDE_STREAMS[key]


class Detector(nn.Module):
    """base of the model nets: __init__ calls the subclass's build() (which creates the modules in the reference's order, so a seeded
    build draws the reference's parameters), then applies cf.weight_init"""

    def __init__(self, cf, logger=None):
        super().__init__()
        self.cf = cf
        self.logger = logger
        self.build()
        if getattr(cf, 'weight_init', None) is not None:
            if logger is not None:
                logger.info("using pytorch weight init of type {}".format(cf.weight_init))
            mutils.initialize_weights(self)
        elif logger is not None:
            logger.info("using default pytorch weight init")

    def _check_patch_size(self, check_z=False):
        h, w = self.cf.patch_size[:2]
        if h / 2 ** 5 != int(h / 2 ** 5) or w / 2 ** 5 != int(w / 2 ** 5):
            raise Exception("Image size must be dividable by 2 at least 5 times to avoid fractions when downscaling and upscaling.")
        if check_z and len(self.cf.patch_size) == 3:
            d = self.cf.patch_size[2]
            if d / 2 ** 3 != int(d / 2 ** 3):
                raise Exception("Image z dimension must be dividable by 2 at least 3 times to avoid fractions when downscaling and upscaling.")

    def _register_anchors(self):
        """np_anchors (numpy, for the monitoring boxes), anchors (fp32, box decoding) and anchors_f64 (the matching kernels)"""
        self.np_anchors = mutils.generate_pyramid_anchors(self.logger, self.cf)
        self.register_buffer("anchors", torch.from_numpy(self.np_anchors).float(), persistent=False)
        self.register_buffer("anchors_f64", torch.from_numpy(self.np_anchors).double(), persistent=False)

    def _to_device(self, arr, dtype=torch.float32):
        """host batch array -> device through pinned memory (non_blocking H2D)"""
        dev = next(self.parameters()).device
        if torch.is_tensor(arr):
            return arr.to(dev, dtype=dtype, non_blocking=True)
        t = torch.from_numpy(np.ascontiguousarray(arr))
        if dev.type == 'cuda':
            t = t.pin_memory()
        return t.to(dev, non_blocking=True).to(dtype)

    # the process group of parallel.sync_batch_statistics (None: every statistic is per rank)
    sync_group = None

    def seg_loss_group(self):
        """the group the seg loss is taken over: sync_group in training mode, None (per rank) in eval mode"""
        return self.sync_group if self.training else None

    def _seg_to_device(self, seg, fused_losses):
        """label map (b, 1, y, x, (z)) -> device: uint8 (1 byte per voxel over PCIe) for the fused seg loss, int64 for the torch-op one"""
        fused = fused_losses and next(self.parameters()).is_cuda and self.cf.num_seg_classes <= 8
        return self._to_device(seg, dtype=torch.uint8 if fused else torch.long)

    def _to_host(self, tensors):
        """device tensors -> numpy through cached pinned staging buffers: all copies are queued, then ONE synchronisation"""
        outs = []
        for i, t in enumerate(tensors):
            t = t.detach().contiguous()
            key = (id(self), i, tuple(t.shape), t.dtype)
            buf = _PINNED.get(key)
            if buf is None:
                buf = torch.empty(t.shape, dtype=t.dtype, pin_memory=t.is_cuda)
                _PINNED[key] = buf
            buf.copy_(t, non_blocking=True)
            outs.append(buf)
        if tensors and tensors[0].is_cuda:
            torch.cuda.current_stream(tensors[0].device).synchronize()
        return [o.numpy().copy() for o in outs]


def match_anchors(net, batch_gt_boxes, batch_gt_class_ids, box_results_list, dev, class_agnostic=False):
    """appends the GT boxes to box_results_list and matches them to net's anchors per batch element -> [(matches int32 [A], target deltas
    float64 [T, 2*dim], positive anchor ids int64)].  class_agnostic: match without the class ids (the RPN's foreground / background).

    The matching synchronises with the host (exact-length positive lists, numpy sub-sampling), so it runs before the network is queued, on a
    side stream: those waits then cover only the matching kernels, and the host is not held up by — nor the GPU drained of — the previous
    step's backward pass still in flight."""
    main_stream = torch.cuda.current_stream(dev) if dev.type == 'cuda' else None
    match_stream = _side_stream(dev) if main_stream is not None else None
    matched = []
    with (torch.cuda.stream(match_stream) if main_stream is not None else contextlib.nullcontext()):
        for b, gt_boxes in enumerate(batch_gt_boxes):
            for ix in range(len(gt_boxes)):
                box_results_list[b].append({'box_coords': gt_boxes[ix], 'box_label': batch_gt_class_ids[b][ix], 'box_type': 'gt'})
            matched.append(mutils.gt_anchor_matching_device(net.cf, net.anchors_f64, gt_boxes, None if class_agnostic else batch_gt_class_ids[b],
                                                            return_pos=True))
    if main_stream is not None:
        main_stream.wait_stream(match_stream)              # the losses (main stream) consume the matching's tensors
        for tup in matched:
            for t in tup:
                t.record_stream(main_stream)
    return matched


def anchor_losses(matched, class_logits, pred_deltas, cf, class_loss_fn, bbox_loss_fn):
    """batch means of the per-element anchor class and box losses -> (class_loss [1], bbox_loss [1], [(matches, sampled negative ids)] for
    append_anchor_boxes).  class_loss_fn(matches, logits, max_pos=, pos_ids=) -> (loss, neg_ix); bbox_loss_fn(target_deltas, pred_deltas,
    matches, max_pos=, pos_ids=) -> loss."""
    n_b = len(matched)
    max_pos = max(1, cf.rpn_train_anchors_per_image // 2)
    class_loss = class_logits.new_zeros(1, dtype=torch.float32)
    bbox_loss = class_logits.new_zeros(1, dtype=torch.float32)
    monitor = []
    for b, (match, target_deltas, pos_ids) in enumerate(matched):
        cl, neg_ix = class_loss_fn(match, class_logits[b], max_pos=max_pos, pos_ids=pos_ids)
        bl = bbox_loss_fn(target_deltas, pred_deltas[b], match, max_pos=max_pos, pos_ids=pos_ids)
        class_loss = class_loss + cl / n_b
        bbox_loss = bbox_loss + bl / n_b
        monitor.append((match, neg_ix))
    return class_loss, bbox_loss, monitor


def seg_loss_terms(seg_logits, seg, cf, group=None):
    """-> (1 - soft dice, cross-entropy) of the seg logits against the label map (b, 1, y, x, (z)).  uint8 labels (Detector._seg_to_device):
    one pass over the logits and the labels each way in the fused kernel (csrc/loss_ops.cu), no one-hot / probability volumes; int64 labels:
    the formulation in torch ops.  group: take both terms over the batch of all its ranks (fused kernel only)."""
    if seg.dtype == torch.uint8:
        dice_score, seg_ce = native_ops.seg_loss(seg_logits, seg.contiguous(), group=group)
        return 1 - dice_score, seg_ce
    if group is not None:
        raise RuntimeError("seg_loss_terms: the seg loss over a process group runs on the fused kernel only (uint8 labels, <= 8 classes)")
    seg_ohe = F.one_hot(seg[:, 0], cf.num_seg_classes).movedim(-1, 1).float()  # on-device one-hot (reference: numpy)
    return 1 - mutils.batch_dice(F.softmax(seg_logits, dim=1), seg_ohe), F.cross_entropy(seg_logits, seg[:, 0])


def append_anchor_boxes(np_anchors, host_matches, host_neg_ix, spatial, dim, box_results_list):
    """positive / sampled-negative anchors of the anchor loss for the monitoring plots, from host copies of each element's matches and
    neg_ix (indices into the element's negative anchors, padded with -1)"""
    hi = np.array([spatial[0], spatial[1], spatial[0], spatial[1]] + ([spatial[2], spatial[2]] if dim == 3 else []))
    for b, (m, nix) in enumerate(zip(host_matches, host_neg_ix)):
        for p in np.clip(np_anchors[m > 0], 0, hi):
            box_results_list[b].append({'box_coords': p, 'box_type': 'pos_anchor'})
        neg_all = np.where(m == -1)[0]
        if neg_all.size:
            for n in np.clip(np_anchors[neg_all[nix[nix >= 0]]], 0, hi):
                box_results_list[b].append({'box_coords': n, 'box_type': 'neg_anchor'})
