"""Torch-facing wrappers of the native ops (NMS, RoIAlign) of libmdt_b200.so.

Reference call surface mirrored (paths relative to the reference root):
  cuda_functions/nms_3D/pth_nms.py:5-17                                 nms_gpu(dets, thresh) -> LongTensor keep (cuda)
  cuda_functions/roi_align_3D/roi_align/crop_and_resize.py:10-69        CropAndResizeFunction / CropAndResize
"""
import ctypes

import torch

from . import _lib as L
from . import parallel as P


def nms_sorted(dets_sorted, thresh, dim):
    """Greedy NMS on boxes ALREADY sorted by descending score, entirely on the device.

    dets_sorted: [N, 2*dim+1] f32 cuda contiguous.  Returns (keep[N] int64 — first num entries valid, num[1] int32), both on the
    device, no host synchronisation (the reduction of nms_cuda.c:33-61 runs in a kernel).
    """
    L.require_cuda(dets_sorted)
    lib = L.load()
    if dets_sorted.dtype != torch.float32 or dets_sorted.dim() != 2 or dets_sorted.shape[1] != 2 * dim + 1:
        raise L.MdtError("nms: dets must be float32 [N, %d]" % (2 * dim + 1))
    if not dets_sorted.is_contiguous():
        raise L.MdtError("nms: boxes must be contiguous")  # same check as nms_cuda.c:19-20
    n = dets_sorted.shape[0]
    dev = dets_sorted.device
    keep = torch.empty(n, dtype=torch.int64, device=dev)
    num = torch.empty(1, dtype=torch.int32, device=dev)
    ws_bytes = lib.mdt_nms_workspace_bytes(n)
    ws = torch.empty(max(ws_bytes, 8), dtype=torch.uint8, device=dev)
    fn = lib.mdt_nms_3d if dim == 3 else lib.mdt_nms_2d
    with torch.cuda.device(dev):
        L.check(fn(L.ptr(dets_sorted), n, float(thresh), L.ptr(ws), ws_bytes, L.ptr(keep), L.ptr(num), L.stream_ptr()))
    return keep, num


def nms_gpu(dets, thresh, dim=None):
    """Drop-in for pth_nms.nms_gpu: sort by the last column (descending), NMS, return indices into `dets` in descending-score order."""
    if dim is None:
        dim = (dets.shape[1] - 1) // 2
    L.require_cuda(dets)
    if dets.shape[0] == 0:
        return torch.empty(0, dtype=torch.int64, device=dets.device)
    scores = dets[:, -1]
    order = scores.sort(0, descending=True)[1]
    keep, num = nms_sorted(dets[order].contiguous().float(), thresh, dim)
    return order[keep[: int(num.item())]].contiguous()  # the one sync the reference API shape requires (exact-length result)


def nms_mask(dets_sorted, thresh, dim):
    """Suppression bit-matrix [N, ceil(N/64)] (as int64 words), the contract of the reference's `_nms` (nms_kernel.h:11-12)."""
    L.require_cuda(dets_sorted)
    lib = L.load()
    n = dets_sorted.shape[0]
    cb = (n + 63) // 64
    mask = torch.empty((n, cb), dtype=torch.int64, device=dets_sorted.device)
    fn = lib.mdt_nms_mask_3d if dim == 3 else lib.mdt_nms_mask_2d
    with torch.cuda.device(dets_sorted.device):
        L.check(fn(n, L.ptr(dets_sorted.contiguous()), L.ptr(mask), float(thresh), L.stream_ptr()))
    return mask


def _strides5(t, dim):
    """element strides of a logical [N, C, (spatial...)] tensor; 2D tensors are [N, C, H, W]"""
    return L.i64arr(list(t.stride()))


class _CropAndResize(torch.autograd.Function):
    """static autograd.Function behind the reference's legacy instance-style Function (crop_and_resize.py:10-51)"""

    @staticmethod
    def forward(ctx, image, boxes, box_ind, crop_size, channels_last_out):
        L.require_cuda(image, boxes, box_ind)
        lib = L.load()
        dim = len(crop_size)
        if image.dim() != dim + 2:
            raise L.MdtError("crop_and_resize: image must be [B, C, %s]" % ("Y, X, Z" if dim == 3 else "Y, X"))
        if image.dtype != torch.float32:
            raise L.MdtError("crop_and_resize: image must be float32")
        boxes = boxes.detach().contiguous().float()
        box_ind = box_ind.detach().contiguous().int()
        n = boxes.shape[0]
        B, C = image.shape[0], image.shape[1]
        sp = list(image.shape[2:])
        out_shape = [n, C] + list(crop_size)
        if channels_last_out and dim == 3:
            crops = torch.empty(out_shape, dtype=torch.float32, device=image.device, memory_format=torch.channels_last_3d)
        elif channels_last_out and dim == 2:
            crops = torch.empty(out_shape, dtype=torch.float32, device=image.device, memory_format=torch.channels_last)
        else:
            crops = torch.empty(out_shape, dtype=torch.float32, device=image.device)
        img = image.detach()
        with torch.cuda.device(image.device):
            if dim == 3:
                L.check(lib.mdt_crop_and_resize_3d_forward(L.ptr(img), L.i64arr(img.stride()), L.ptr(boxes), L.ptr(box_ind), n, B, sp[0], sp[1], sp[2],
                                                           crop_size[0], crop_size[1], crop_size[2], C, 0.0, L.ptr(crops),
                                                           L.i64arr(crops.stride()), L.stream_ptr()))
            else:
                L.check(lib.mdt_crop_and_resize_2d_forward(L.ptr(img), L.i64arr(img.stride()), L.ptr(boxes), L.ptr(box_ind), n, B, sp[0], sp[1],
                                                           crop_size[0], crop_size[1], C, 0.0, L.ptr(crops), L.i64arr(crops.stride()),
                                                           L.stream_ptr()))
        ctx.save_for_backward(boxes, box_ind)
        ctx.im_size = tuple(image.shape)
        ctx.im_strides = tuple(image.stride())
        ctx.crop_size = tuple(crop_size)
        return crops

    @staticmethod
    def backward(ctx, grad_out):
        boxes, box_ind = ctx.saved_tensors
        lib = L.load()
        dim = len(ctx.crop_size)
        B, C = ctx.im_size[0], ctx.im_size[1]
        sp = ctx.im_size[2:]
        # gradient gets the memory layout of the forward image (dense tensors only)
        grad_image = torch.empty_strided(ctx.im_size, ctx.im_strides, dtype=torch.float32, device=grad_out.device)
        dense = grad_image.numel() == _storage_extent(ctx.im_size, ctx.im_strides)
        if not dense:
            grad_image = torch.empty(ctx.im_size, dtype=torch.float32, device=grad_out.device)
        g = grad_out.detach().float()
        if not (g.is_contiguous() or g.is_contiguous(memory_format=torch.channels_last_3d if dim == 3 else torch.channels_last)):
            g = g.contiguous()
        n = boxes.shape[0]
        with torch.cuda.device(grad_out.device):
            if dim == 3:
                L.check(lib.mdt_crop_and_resize_3d_backward(L.ptr(g), L.i64arr(g.stride()), L.ptr(boxes), L.ptr(box_ind), n, B, sp[0], sp[1], sp[2],
                                                            ctx.crop_size[0], ctx.crop_size[1], ctx.crop_size[2], C, L.ptr(grad_image),
                                                            L.i64arr(grad_image.stride()), 1, grad_image.numel(), L.stream_ptr()))
            else:
                L.check(lib.mdt_crop_and_resize_2d_backward(L.ptr(g), L.i64arr(g.stride()), L.ptr(boxes), L.ptr(box_ind), n, B, sp[0], sp[1],
                                                            ctx.crop_size[0], ctx.crop_size[1], C, L.ptr(grad_image),
                                                            L.i64arr(grad_image.stride()), 1, grad_image.numel(), L.stream_ptr()))
        return grad_image, None, None, None, None


class _PyramidRoIAlign(torch.autograd.Function):
    """RoIAlign of every RoI on its own pyramid level in ONE kernel launch (mdt_pyramid_roi_align_{forward,backward}); gradient to the maps"""

    @staticmethod
    def forward(ctx, boxes, box_ind, roi_level, crop_size, *maps):
        lib = L.load()
        L.require_cuda(boxes, box_ind, roi_level, *maps)
        dim = len(crop_size)
        mf = torch.channels_last_3d if dim == 3 else torch.channels_last
        maps = [m.contiguous(memory_format=mf) for m in maps]
        B, C = maps[0].shape[0], maps[0].shape[1]
        n = boxes.shape[0]
        boxes = boxes.detach().contiguous().float()
        box_ind = box_ind.contiguous().int()
        roi_level = roi_level.contiguous().int()
        crops = torch.empty((n, C) + tuple(crop_size), dtype=torch.float32, device=boxes.device).contiguous(memory_format=mf)
        nl = len(maps)
        ptrs = (ctypes.c_void_p * nl)(*[m.data_ptr() for m in maps])
        strides = L.i64arr([s for m in maps for s in (tuple(m.stride()) + (0,) * (5 - m.dim()))])
        dims = (ctypes.c_int * (3 * nl))(*[d for m in maps for d in (tuple(m.shape[2:]) + (1,) * (5 - m.dim()))])
        cz = crop_size[2] if dim == 3 else 1
        with torch.cuda.device(boxes.device):
            rc = lib.mdt_pyramid_roi_align_forward(dim, ptrs, strides, dims, nl, L.ptr(boxes), L.ptr(box_ind), L.ptr(roi_level), n, B, crop_size[0],
                                                   crop_size[1], cz, C, L.ptr(crops), L.i64arr(tuple(crops.stride()) + (0,) * (5 - crops.dim())),
                                                   L.stream_ptr())
        L.check(rc)
        ctx.save_for_backward(boxes, box_ind, roi_level)
        ctx.meta = (tuple(crop_size), [tuple(m.shape) for m in maps], [tuple(m.stride()) for m in maps], dim)
        return crops

    @staticmethod
    def backward(ctx, grad_out):
        boxes, box_ind, roi_level = ctx.saved_tensors
        crop_size, shapes, strides_, dim = ctx.meta
        lib = L.load()
        mf = torch.channels_last_3d if dim == 3 else torch.channels_last
        g = grad_out.detach().float().contiguous(memory_format=mf)
        grads = [torch.empty_strided(sh, st, dtype=torch.float32, device=g.device) for sh, st in zip(shapes, strides_)]
        nl = len(grads)
        ptrs = (ctypes.c_void_p * nl)(*[m.data_ptr() for m in grads])
        strides = L.i64arr([s for st in strides_ for s in (tuple(st) + (0,) * (5 - len(st)))])
        dims = (ctypes.c_int * (3 * nl))(*[d for sh in shapes for d in (tuple(sh[2:]) + (1,) * (5 - len(sh)))])
        numel = L.i64arr([m.numel() for m in grads])
        cz = crop_size[2] if dim == 3 else 1
        with torch.cuda.device(g.device):
            L.check(lib.mdt_pyramid_roi_align_backward(dim, L.ptr(g), L.i64arr(tuple(g.stride()) + (0,) * (5 - g.dim())), L.ptr(boxes), L.ptr(box_ind),
                                                       L.ptr(roi_level), boxes.shape[0], shapes[0][0], crop_size[0], crop_size[1], cz, shapes[0][1], ptrs,
                                                       strides, dims, nl, 1, numel, L.stream_ptr()))
        return (None, None, None, None) + tuple(grads)


def pyramid_roi_align(maps, boxes, box_ind, roi_level, crop_size):
    """crops [n, C, *crop_size] (channels-last) of RoI n taken from maps[roi_level[n]]; one launch; falls back to per-level launches (summed,
    rows of other levels are zero) when a map layout is outside the vector kernel"""
    try:
        return _PyramidRoIAlign.apply(boxes, box_ind, roi_level, tuple(int(c) for c in crop_size), *maps)
    except L.MdtError as e:
        if "unsupported" not in str(e).lower():
            raise
    fn = (CropAndResizeFunction if len(crop_size) == 3 else CropAndResizeFunction2D)(*crop_size, 0)
    out = None
    for lv, m in enumerate(maps):
        ind = torch.where(roi_level == lv, box_ind, box_ind.new_full((), -1))
        y = fn(m, boxes, ind)
        out = y if out is None else out + y
    return out


def _storage_extent(size, stride):
    ext = 1
    for s, st in zip(size, stride):
        if s == 0:
            return 0
        ext += (s - 1) * st
    return ext


class CropAndResizeFunction(object):
    """Callable with the reference's construction/call shape:  CropAndResizeFunction(ch, cw[, cz], extrapolation_value)(image, boxes, box_ind).

    2D form takes (crop_height, crop_width, extrapolation_value=0), 3D form (crop_height, crop_width, crop_zdepth, extrapolation_value=0)
    (roi_align_2D/roi_align/crop_and_resize.py vs roi_align_3D/roi_align/crop_and_resize.py).  extrapolation_value is accepted and
    unused, exactly as in the reference GPU kernel.  Gradient flows to `image` only (crop_and_resize.py:51).
    Output layout follows the image: a channels-last image yields channels-last crops (logical shape is always [n, C, ch, cw(, cz)]).
    """
    dim = 3

    def __init__(self, crop_height, crop_width, *rest):
        if self.dim == 3:
            if len(rest) < 1:
                raise TypeError("3D CropAndResizeFunction needs crop_zdepth")
            self.crop_size = (int(crop_height), int(crop_width), int(rest[0]))
            self.extrapolation_value = rest[1] if len(rest) > 1 else 0
        else:
            self.crop_size = (int(crop_height), int(crop_width))
            self.extrapolation_value = rest[0] if len(rest) > 0 else 0

    def __call__(self, image, boxes, box_ind):
        cl = image.stride(1) == 1 and image.shape[1] > 1
        return _CropAndResize.apply(image, boxes, box_ind, self.crop_size, cl)

    # legacy spelling used by some callers
    forward = __call__


class CropAndResizeFunction2D(CropAndResizeFunction):
    dim = 2


class CropAndResize(torch.nn.Module):
    """nn.Module twin (crop_and_resize.py:54-69)"""
    _fn = CropAndResizeFunction

    def __init__(self, *args):
        super().__init__()
        self.fn = self._fn(*args)

    def forward(self, image, boxes, box_ind):
        return self.fn(image, boxes, box_ind)


class CropAndResize2D(CropAndResize):
    _fn = CropAndResizeFunction2D


# ------------------------------------------------------------------------------------------------------------------ loss-side kernels
def _seg_layout(logits):
    """(batch, class, voxel) element strides of a [b, c, spatial...] logit map whose spatial axes collapse to one stride; None otherwise"""
    sp = logits.shape[2:]
    st = logits.stride()
    sv = st[-1]
    run = sv
    for size, stride in zip(reversed(sp), reversed(st[2:])):
        if size != 1 and stride != run:
            return None
        run *= size
    return st[0], st[1], sv


def _seg_loss_args(logits, target, class_weights):
    """-> (logits with a collapsible layout, its (batch, class, voxel) strides, n, classes, voxels) after the checks both seg-loss paths share"""
    lay = _seg_layout(logits)
    if lay is None:
        logits = logits.contiguous()
        lay = _seg_layout(logits)
    n, c = logits.shape[0], logits.shape[1]
    vox = 1
    for s in logits.shape[2:]:
        vox *= s
    if target.dtype != torch.uint8 or target.numel() != n * vox or not target.is_contiguous():
        raise L.MdtError("seg_loss: target must be a contiguous uint8 label map with one entry per voxel")
    if class_weights is not None:
        if class_weights.dtype != torch.float32 or class_weights.numel() != c or not class_weights.is_contiguous():
            raise L.MdtError("seg_loss: class_weights must be a contiguous float32 tensor with one weight per class")
        if class_weights.device != logits.device:
            raise L.MdtError("seg_loss: class_weights must be on the logits' device (%s), got %s" % (logits.device, class_weights.device))
    return logits, lay, n, c, vox


class _SegLoss(torch.autograd.Function):
    """(dice score over the batch pseudo-volume, mean voxel cross-entropy) of seg logits vs a uint8 label map, csrc/loss_ops.cu — replaces
    softmax + one-hot + batch_dice + cross_entropy (retina_unet.py:395,446-448; model_utils.py:785-799,833-858) by one pass each way"""

    @staticmethod
    def forward(ctx, logits, target, fpw, smooth, class_weights):
        L.require_cuda(logits, target, class_weights)
        lib = L.load()
        logits, lay, n, c, vox = _seg_loss_args(logits, target, class_weights)
        dev = logits.device
        sums = torch.empty(3 * c + 1, dtype=torch.float64, device=dev)
        out = torch.empty(2, dtype=torch.float32, device=dev)
        ws_bytes = lib.mdt_seg_loss_workspace_bytes(c)
        if ws_bytes == 0:
            raise L.MdtError("seg_loss: at most 8 classes")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        strides = L.i64arr(lay)
        with torch.cuda.device(dev):
            if class_weights is None:
                L.check(lib.mdt_seg_loss_forward(L.ptr(logits), strides, L.ptr(target), n, vox, c, float(fpw), float(smooth), L.ptr(sums), L.ptr(out),
                                                 L.ptr(ws), ws_bytes, L.stream_ptr()))
            else:
                L.check(lib.mdt_seg_loss_weighted_forward(L.ptr(logits), strides, L.ptr(target), n, vox, c, float(fpw), float(smooth), L.ptr(class_weights),
                                                          L.ptr(sums), L.ptr(out), L.ptr(ws), ws_bytes, L.stream_ptr()))
        ctx.save_for_backward(logits, target, sums, class_weights)
        ctx.meta = (lay, n, vox, c, float(fpw), float(smooth))
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_dice, g_ce):
        lib = L.load()
        logits, target, sums, class_weights = ctx.saved_tensors
        lay, n, vox, c, fpw, smooth = ctx.meta
        zero = logits.new_zeros(())                      # an output that did not enter the loss arrives as None
        gout = torch.stack([(g_dice if g_dice is not None else zero).reshape(()), (g_ce if g_ce is not None else zero).reshape(())]).to(torch.float32).contiguous()
        grad = torch.empty_strided(logits.shape, logits.stride(), dtype=torch.float32, device=logits.device)
        with torch.cuda.device(logits.device):
            if class_weights is None:
                L.check(lib.mdt_seg_loss_backward(L.ptr(logits), L.i64arr(lay), L.ptr(target), n, vox, c, fpw, smooth, L.ptr(sums), L.ptr(gout), L.ptr(grad),
                                                  L.stream_ptr()))
            else:
                L.check(lib.mdt_seg_loss_weighted_backward(L.ptr(logits), L.i64arr(lay), L.ptr(target), n, vox, c, fpw, smooth, L.ptr(class_weights),
                                                           L.ptr(sums), L.ptr(gout), L.ptr(grad), L.stream_ptr()))
        return grad, None, None, None, None


class _SyncSegLoss(torch.autograd.Function):
    """_SegLoss over the batch of all ranks of `group` (the same n on every rank): per-sample sums -> one exchange -> dice and CE of the whole
    batch on every rank.  Each rank's loss holds the global term once, so the backward sums the incoming gradients over the ranks (the SyncBN
    rule, done by gathering every rank's incoming pair and adding the pairs in rank order in the kernel): after FlatGradAllReduce averages the
    parameter gradients, they are the one-GPU gradients of that term."""

    @staticmethod
    def forward(ctx, logits, target, fpw, smooth, class_weights, group):
        L.require_cuda(logits, target, class_weights)
        lib = L.load()
        logits, lay, n, c, vox = _seg_loss_args(logits, target, class_weights)
        dev = logits.device
        ws_bytes = lib.mdt_seg_loss_sample_workspace_bytes(n, vox, c)
        if ws_bytes == 0:
            raise L.MdtError("seg_loss: at most 8 classes")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        sums = torch.empty(3 * c + 1, dtype=torch.float64, device=dev)
        out = torch.empty(2, dtype=torch.float32, device=dev)
        strides = L.i64arr(lay)
        with torch.cuda.device(dev):
            buf, slot = P.row_slots(n, 3 * c + 1, dev, group)
            if class_weights is None:
                L.check(lib.mdt_seg_loss_sample_sums(L.ptr(logits), strides, L.ptr(target), n, vox, c, L.ptr(slot), L.ptr(ws), ws_bytes, L.stream_ptr()))
            else:
                L.check(lib.mdt_seg_loss_weighted_sample_sums(L.ptr(logits), strides, L.ptr(target), n, vox, c, L.ptr(class_weights), L.ptr(slot),
                                                              L.ptr(ws), ws_bytes, L.stream_ptr()))
            rows = P.all_reduce_rows(buf, group)
            L.check(lib.mdt_seg_loss_from_sums(L.ptr(rows), rows.shape[0], vox, c, float(fpw), float(smooth), L.ptr(class_weights), L.ptr(sums),
                                               L.ptr(out), L.stream_ptr()))
        ctx.save_for_backward(logits, target, sums, class_weights)
        ctx.meta = (lay, n, vox, c, float(fpw), float(smooth), rows.shape[0] * vox, group)
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_dice, g_ce):
        lib = L.load()
        logits, target, sums, class_weights = ctx.saved_tensors
        lay, n, vox, c, fpw, smooth, total, group = ctx.meta
        zero = logits.new_zeros(())                      # an output that did not enter the loss arrives as None
        grad = torch.empty_strided(logits.shape, logits.stride(), dtype=torch.float32, device=logits.device)
        with torch.cuda.device(logits.device):
            # every rank's {dL/d dice, dL/d ce} in rank order: the kernel adds them in fp64 in that order
            buf, slot = P.row_slots(1, 2, logits.device, group, dtype=torch.float32)
            torch.stack([(g if g is not None else zero).reshape(()) for g in (g_dice, g_ce)], out=slot[0])
            gout = P.all_reduce_rows(buf, group)
            if class_weights is None:
                L.check(lib.mdt_seg_loss_backward_global(L.ptr(logits), L.i64arr(lay), L.ptr(target), n, vox, c, fpw, smooth, L.ptr(sums), total,
                                                         L.ptr(gout), gout.shape[0], L.ptr(grad), L.stream_ptr()))
            else:
                L.check(lib.mdt_seg_loss_weighted_backward_global(L.ptr(logits), L.i64arr(lay), L.ptr(target), n, vox, c, fpw, smooth, L.ptr(class_weights),
                                                                  L.ptr(sums), total, L.ptr(gout), gout.shape[0], L.ptr(grad), L.stream_ptr()))
        return grad, None, None, None, None, None


def seg_loss(seg_logits, seg_labels_u8, false_positive_weight=1.0, smooth=1e-6, class_weights=None, group=None):
    """-> (batch_dice(softmax(seg_logits), one_hot(labels)), cross_entropy(seg_logits, labels)), both differentiable 0-d tensors.
    class_weights: optional per-class weights of the cross-entropy on the logits' device (F.cross_entropy(weight=)); the dice term is unchanged.
    group: a process group whose ranks hold the rest of the batch (the same batch size on every rank): dice and CE are then those of the whole
    batch, in rank order, on every rank, and every rank must run this loss's backward"""
    if seg_logits.dtype != torch.float32:
        raise L.MdtError("seg_loss: logits must be float32")
    if group is not None:
        return _SyncSegLoss.apply(seg_logits, seg_labels_u8, false_positive_weight, smooth, class_weights, group)
    return _SegLoss.apply(seg_logits, seg_labels_u8, false_positive_weight, smooth, class_weights)


SEG_COMPONENTS_MAX_K = 128


def seg_components(seg_logits, n_fg_classes, k, median=False, return_labels=False):
    """Connected-component boxes of the argmax of softmax(seg_logits) (the reference's detection_unet forward + get_coords), on the device, no sync.

    seg_logits: fp32 [b, S, y, x(, z)], S <= 8, any layout whose spatial axes collapse to one stride (NCDHW or channels-last).
    -> dict: seg_pred uint8 [b, y, x(, z)]; boxes int32 [b, n_fg_classes, k, 2*dim]; scores f32 [b, n_fg_classes, k]; n_kept int32
    [b, n_fg_classes]; labels int32 [b, y, x(, z)] (dense component id in scipy's label order, -1 background) when return_labels.
    Components per (element, class): the k largest by voxel count (ties: larger label first); score = max (or exact median) probability."""
    L.require_cuda(seg_logits)
    lib = L.load()
    if seg_logits.dtype != torch.float32 or seg_logits.dim() not in (4, 5):
        raise L.MdtError("seg_components: logits must be float32 [b, classes, y, x(, z)]")
    dim = seg_logits.dim() - 2
    lay = _seg_layout(seg_logits)
    if lay is None:
        seg_logits = seg_logits.contiguous()
        lay = _seg_layout(seg_logits)
    b, S = seg_logits.shape[0], seg_logits.shape[1]
    sp = tuple(seg_logits.shape[2:])
    y, x, z = sp[0], sp[1], (sp[2] if dim == 3 else 1)
    ws_bytes = lib.mdt_seg_components_workspace_bytes(b, y, x, z, S, int(n_fg_classes), int(k), dim)
    if ws_bytes == 0:
        raise L.MdtError("seg_components: unsupported arguments (at most 8 classes, 1 <= k <= %d, fewer than 2^31 voxels)" % SEG_COMPONENTS_MAX_K)
    dev = seg_logits.device
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    seg_pred = torch.empty((b,) + sp, dtype=torch.uint8, device=dev)
    labels = torch.empty((b,) + sp, dtype=torch.int32, device=dev) if return_labels else None
    boxes = torch.empty((b, n_fg_classes, k, 2 * dim), dtype=torch.int32, device=dev)
    scores = torch.empty((b, n_fg_classes, k), dtype=torch.float32, device=dev)
    n_kept = torch.empty((b, n_fg_classes), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.mdt_seg_components(L.ptr(seg_logits.detach()), L.i64arr(lay), b, y, x, z, S, int(n_fg_classes), int(k), dim, int(bool(median)),
                                       L.ptr(seg_pred), L.ptr(labels), L.ptr(boxes), L.ptr(scores), L.ptr(n_kept), L.ptr(ws), ws_bytes, L.stream_ptr()))
    out = {'seg_pred': seg_pred, 'boxes': boxes, 'scores': scores, 'n_kept': n_kept}
    if return_labels:
        out['labels'] = labels
    return out


SHEM_MAX_POOL = 1024


def shem_supported(logits, k_pos, k_pool):
    return (logits.is_cuda and logits.dtype == torch.float32 and logits.dim() == 2 and 2 <= logits.shape[1] <= 8 and 1 <= k_pos <= SHEM_MAX_POOL
            and 1 <= k_pool <= SHEM_MAX_POOL)


class _ShemClassLoss(torch.autograd.Function):
    """fused class loss with stochastic hard-example mining (csrc/loss_ops.cu); see retina_unet.compute_class_loss for the semantics"""

    @staticmethod
    def forward(ctx, logits, matches, pos_ids, rand_keys, k_pos, k_pool, k_neg, poolsize):
        L.require_cuda(logits, matches, rand_keys)
        lib = L.load()
        logits = logits.contiguous()
        a, c = logits.shape
        dev = logits.device
        matches = matches.to(torch.int32).contiguous()
        pos_ids = pos_ids.to(torch.int64).contiguous()
        rand_keys = rand_keys.to(torch.float32).contiguous()
        if rand_keys.numel() != k_pool:
            raise L.MdtError("shem: rand_keys must hold k_pool entries")
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        neg_ix = torch.empty(k_neg, dtype=torch.int64, device=dev)
        rows = torch.empty(k_pos + k_neg, dtype=torch.int32, device=dev)
        labels = torch.empty(k_pos + k_neg, dtype=torch.int32, device=dev)
        w = torch.empty(k_pos + k_neg, dtype=torch.float32, device=dev)
        ws_bytes = lib.mdt_shem_workspace_bytes(a, k_pool)
        ws = torch.empty(max(ws_bytes, 8), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.mdt_shem_class_loss_forward(L.ptr(logits), L.ptr(matches), a, c, L.ptr(pos_ids) if pos_ids.numel() else None, int(pos_ids.numel()),
                                                    k_pos, k_pool, k_neg, poolsize, L.ptr(rand_keys), L.ptr(loss), L.ptr(neg_ix), L.ptr(rows), L.ptr(labels),
                                                    L.ptr(w), L.ptr(ws), ws_bytes, L.stream_ptr()))
        ctx.save_for_backward(logits, rows, labels, w)
        ctx.mark_non_differentiable(neg_ix)
        return loss[0], neg_ix

    @staticmethod
    def backward(ctx, g_loss, _g_neg):
        lib = L.load()
        logits, rows, labels, w = ctx.saved_tensors
        a, c = logits.shape
        grad = torch.empty_like(logits)
        g = g_loss.reshape(1).to(torch.float32).contiguous()
        with torch.cuda.device(logits.device):
            L.check(lib.mdt_shem_class_loss_backward(L.ptr(logits), a, c, L.ptr(rows), L.ptr(labels), L.ptr(w), int(rows.numel()), L.ptr(g), L.ptr(grad),
                                                     L.stream_ptr()))
        return grad, None, None, None, None, None, None, None


def shem_class_loss(logits, matches, pos_ids, rand_keys, k_pos, k_pool, k_neg, poolsize):
    """-> (loss 0-d, neg_ix [k_neg] int64 padded with -1)"""
    return _ShemClassLoss.apply(logits, matches, pos_ids, rand_keys, int(k_pos), int(k_pool), int(k_neg), int(poolsize))


def unmold_masks(detections, detection_masks, img_shape, want_float=False):
    """Mask R-CNN's full-size segmentation (csrc/unmold.cu): every detection's mask of its class, resized to its box as scipy.ndimage.zoom(order=1)
    does and pasted into the image; per batch element the maximum over the detections, rounded half to even.  No host synchronisation.

    detections: fp32 [n, 2*dim+3] rows (y1, x1, y2, x2, (z1, z2), batch_ix, class_id, score); detection_masks: fp32 [n, C, *mask_shape], any
    strides (the mask head's output is channels-last); img_shape: (b, c, *spatial) or (b, *spatial) with dim spatial axes.
    -> seg uint8 [b, *spatial], and with want_float also the fp32 maximum before rounding [b, *spatial]."""
    L.require_cuda(detections, detection_masks)
    lib = L.load()
    dim = detections.shape[1] - 3 if detections.dim() == 2 else 0
    dim = dim // 2 if dim % 2 == 0 else 0
    if dim not in (2, 3) or detections.dtype != torch.float32 or detection_masks.dtype != torch.float32 or detection_masks.dim() != dim + 2 \
            or detection_masks.shape[0] != detections.shape[0]:
        raise L.MdtError("unmold_masks: detections must be float32 [n, 2*dim+3] and detection_masks float32 [n, C, *mask_shape] with dim 2 or 3")
    spatial = tuple(int(s) for s in img_shape[-dim:])
    b = int(img_shape[0])
    dev = detections.device
    det = detections.detach().contiguous()
    masks = detection_masks.detach()
    n, c = int(det.shape[0]), int(masks.shape[1])
    seg = torch.empty((b,) + spatial, dtype=torch.uint8, device=dev)
    seg_float = torch.empty((b,) + spatial, dtype=torch.float32, device=dev) if want_float else None
    with torch.cuda.device(dev):
        L.check(lib.mdt_unmold_masks(dim, L.ptr(det), n, L.ptr(masks), L.i64arr(masks.stride()), c, (ctypes.c_int * dim)(*masks.shape[2:]), b,
                                     (ctypes.c_int * dim)(*spatial), L.ptr(seg), L.ptr(seg_float), L.stream_ptr()))
    return (seg, seg_float) if want_float else seg
