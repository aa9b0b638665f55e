"""Config objects for the BASELINE.json workloads.  The hot path only READS a `cf` (SURVEY.md Appendix A lists the attributes); these
builders produce one with the values the reference's experiments/lidc_exp/configs.py and experiments/toy_exp/configs.py define for the
named model, so benchmarks and tests run without the reference tree.  Plain attribute bags, like the reference's config classes."""
import types

import numpy as np


def _retina_scales(base):
    return [[s[0], s[0] * (2 ** (1 / 3)), s[0] * (2 ** (2 / 3))] for s in base]


def make_cf(model='retina_unet', dim=3, patch_size=(128, 128, 128), exp='lidc_exp', batch_size=2):
    """model in {'retina_unet', 'retina_net', 'mrcnn', 'ufrcnn', 'detection_unet'}; exp in {'lidc_exp', 'toy_exp'} selects the filter widths,
    the Detection U-Net's n_roi_candidates and UFRCNN+'s sampling sizes, roi_chunk_size and learning-rate schedule length."""
    cf = types.SimpleNamespace()
    cf.dim = dim
    cf.model = model
    cf.n_channels = 1
    cf.patch_size = list(patch_size[:dim])
    cf.batch_size = batch_size
    if exp == 'toy_exp':
        cf.start_filts = 48 if dim == 2 else 18
        cf.end_filts = cf.start_filts * 4 if dim == 2 else cf.start_filts * 2
    else:
        cf.start_filts = 48 if dim == 2 else 18
        cf.end_filts = cf.start_filts * 4 if dim == 2 else cf.start_filts * 2
    cf.res_architecture = 'resnet50'
    cf.norm = None
    cf.relu = 'relu'
    cf.weight_init = None
    cf.sixth_pooling = False
    cf.n_latent_dims = 0
    cf.class_specific_seg_flag = False
    cf.head_classes = 3
    cf.num_seg_classes = 2
    cf.backbone_strides = {'xy': [4, 8, 16, 32], 'z': [1, 2, 4, 8]}
    cf.rpn_anchor_scales = {'xy': [[8], [16], [32], [64]], 'z': [[2], [4], [8], [16]]}
    cf.rpn_anchor_ratios = [0.5, 1, 2]
    cf.rpn_anchor_stride = 1
    cf.pyramid_levels = [0, 1, 2, 3]
    cf.n_rpn_features = 512 if dim == 2 else 128
    cf.rpn_bbox_std_dev = np.array([0.1, 0.1, 0.1, 0.2, 0.2, 0.2])
    cf.bbox_std_dev = np.array([0.1, 0.1, 0.1, 0.2, 0.2, 0.2])
    p = cf.patch_size
    cf.window = np.array([0, 0, p[0], p[1]] + ([0, p[2]] if dim == 3 else []))
    cf.scale = np.array([p[0], p[1], p[0], p[1]] + ([p[2], p[2]] if dim == 3 else []))
    if dim == 2:
        cf.rpn_bbox_std_dev = cf.rpn_bbox_std_dev[:4]
        cf.bbox_std_dev = cf.bbox_std_dev[:4]
    cf.rpn_train_anchors_per_image = 6
    cf.train_rois_per_image = 6
    cf.roi_positive_ratio = 0.5
    cf.anchor_matching_iou = 0.7
    cf.shem_poolsize = 10
    cf.pool_size = (7, 7) if dim == 2 else (7, 7, 3)
    cf.mask_pool_size = (14, 14) if dim == 2 else (14, 14, 5)
    cf.mask_shape = (28, 28) if dim == 2 else (28, 28, 10)
    cf.pre_nms_limit = 3000 if dim == 2 else 6000
    cf.rpn_nms_threshold = 0.7 if dim == 2 else 0.7
    cf.roi_chunk_size = 2500 if dim == 2 else 600
    cf.post_nms_rois_training = 500 if dim == 2 else 75
    cf.post_nms_rois_inference = 500
    cf.model_max_instances_per_batch_element = 10 if dim == 2 else 30
    cf.detection_nms_threshold = 1e-5
    cf.model_min_confidence = 0.1
    cf.operate_stride1 = False
    cf.frcnn_mode = False
    cf.return_masks_in_val = True
    cf.n_plot_rpn_props = 30
    cf.class_dict = {1: 'benign', 2: 'malignant'}
    cf.learning_rate = [1e-4] * 100
    cf.weight_decay = 0.0
    if dim == 2:
        cf.backbone_shapes = np.array([[int(np.ceil(p[0] / s)), int(np.ceil(p[1] / s))] for s in cf.backbone_strides['xy']])
    else:
        cf.backbone_shapes = np.array([[int(np.ceil(p[0] / s)), int(np.ceil(p[1] / s)), int(np.ceil(p[2] / sz))]
                                       for s, sz in zip(cf.backbone_strides['xy'], cf.backbone_strides['z'])])
    if model in ('retina_net', 'retina_unet'):
        cf.rpn_anchor_scales['xy'] = _retina_scales(cf.rpn_anchor_scales['xy'])
        cf.rpn_anchor_scales['z'] = _retina_scales(cf.rpn_anchor_scales['z'])
        cf.n_anchors_per_pos = len(cf.rpn_anchor_ratios) * 3
        cf.n_rpn_features = 256 if dim == 2 else 64
        cf.pre_nms_limit = 10000 if dim == 2 else 50000
        cf.anchor_matching_iou = 0.5
        cf.operate_stride1 = (model == 'retina_unet')
    else:
        cf.n_anchors_per_pos = len(cf.rpn_anchor_ratios)
    if model == 'ufrcnn':
        # add_mrcnn_configs + the `ufrcnn` block of experiments/{lidc_exp,toy_exp}/configs.py, including the values that differ by experiment
        # or dim there and that the other models here take from the lidc_exp 3D config
        cf.operate_stride1 = True
        cf.class_specific_seg_flag = True
        cf.num_seg_classes = 3
        cf.frcnn_mode = True
        cf.return_masks_in_test = False
        cf.n_plot_rpn_props = 5 if dim == 2 else 30
        if exp == 'toy_exp':
            cf.learning_rate = [1e-4] * 24
            cf.rpn_train_anchors_per_image = 2
            cf.train_rois_per_image = 2
            if dim == 2:
                cf.roi_chunk_size = 800
    if model == 'detection_unet':
        # add_det_unet_configs of experiments/{lidc_exp,toy_exp}/configs.py
        cf.aggregation_operation = 'max'
        cf.n_roi_candidates = (3 if dim == 2 else 8) if exp == 'toy_exp' else (10 if dim == 2 else 30)
        cf.seg_loss_mode = 'dice_wce'
        cf.fp_dice_weight = 1
        cf.wce_weights = [1, 1, 1]
        cf.detection_min_confidence = 0.1
        cf.class_specific_seg_flag = True
        cf.num_seg_classes = 3
        cf.head_classes = 3
        cf.operate_stride1 = True
    return cf


def synthetic_batch(cf, batch_size=None, seed=0, with_masks=False):
    """Synthetic patches of the BASELINE shape (SURVEY.md §8d cfg2/cfg3): uniform-noise image, one axis-aligned cuboid ROI per element.
    Keys and formats as produced by the reference's loaders + batchgenerators' ConvertSegToBoundingBoxCoordinates:
    data f32 [B,1,Y,X,(Z)], seg uint8 [B,1,...], bb_target list of [n_roi, 2*dim] int, roi_labels list of [n_roi] int, roi_masks, pid."""
    rs = np.random.RandomState(seed)
    B = batch_size or cf.batch_size
    p = cf.patch_size
    dim = cf.dim
    data = rs.rand(B, cf.n_channels, *p).astype(np.float32)
    seg = np.zeros((B, 1, *p), dtype=np.uint8)
    bb, labels, masks = [], [], []
    for b in range(B):
        size = [int(rs.randint(8, min(33, p[k] // 2 + 1))) for k in range(dim)]
        lo = [int(rs.randint(0, p[k] - size[k] + 1)) for k in range(dim)]
        sl = tuple(slice(lo[k], lo[k] + size[k]) for k in range(dim))
        seg[(b, 0) + sl] = 1
        box = [lo[0], lo[1], lo[0] + size[0], lo[1] + size[1]] + ([lo[2], lo[2] + size[2]] if dim == 3 else [])
        bb.append(np.array([box]))
        labels.append(np.array([int(rs.randint(1, 3))]))
        if with_masks:
            masks.append(seg[b][np.newaxis].copy())
    batch = {'data': data, 'seg': seg, 'bb_target': bb, 'roi_labels': labels, 'pid': ['synth_%d' % i for i in range(B)]}
    if with_masks:
        batch['roi_masks'] = masks
    return batch
