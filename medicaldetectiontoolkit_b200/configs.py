"""Config objects for the BASELINE.json workloads.  The hot path only READS a `cf` (SURVEY.md Appendix A lists the attributes); these
builders produce one with the values the reference's experiments/lidc_exp/configs.py, experiments/toy_exp/configs.py and
experiments/pet_ct_tnm_classification/configs.py define for the named model, so benchmarks and tests run without the reference tree.  Plain
attribute bags, like the reference's config classes."""
import types

import numpy as np


def _retina_scales(base):
    return [[s[0], s[0] * (2 ** (1 / 3)), s[0] * (2 ** (2 / 3))] for s in base]


PETCT = 'pet_ct_tnm_classification'
PETCT_MODELS = ('retina_unet', 'retina_net', 'mrcnn')


def make_cf(model='retina_unet', dim=3, patch_size=None, exp='lidc_exp', batch_size=None):
    """model in {'retina_unet', 'retina_net', 'mrcnn', 'ufrcnn', 'detection_unet'}; exp in {'lidc_exp', 'toy_exp'} selects the filter widths,
    the Detection U-Net's n_roi_candidates and UFRCNN+'s sampling sizes, roi_chunk_size and learning-rate schedule length.  patch_size
    defaults to 128^dim and batch_size to 2.

    exp = 'pet_ct_tnm_classification' (retina_unet, retina_net and mrcnn only) gives that experiment's two input channels (CT + PET), one
    foreground class, its patch (192 x 192 x 32 / 288 x 288) and pre-crop sizes, batch size and learning-rate schedule; its loader converts
    the binary lesion map with get_rois_from_seg_flag=True (augment.Augmenter)."""
    if exp == PETCT:
        if model == 'detection_unet':
            raise ValueError("pet_ct_tnm_classification cannot build detection_unet: its add_det_unet_configs makes a learning-rate schedule of "
                             "75 epochs for num_epochs = 100")
        if model not in PETCT_MODELS:
            raise ValueError("pet_ct_tnm_classification has no %r model (it configures %s)" % (model, ', '.join(PETCT_MODELS)))
        if patch_size is None:
            patch_size = [288, 288] if dim == 2 else [192, 192, 32]
        if batch_size is None:
            batch_size = 20 if dim == 2 else 8
    if patch_size is None:
        patch_size = (128, 128, 128)
    if batch_size is None:
        batch_size = 2
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
    # data augmentation (experiments/lidc_exp/configs.py:156-177; toy_exp/configs.py:163-184 has the same values).  order_data and
    # border_mode_data / border_cval_data are never passed to the SpatialTransform by the reference's loaders (augment.py).
    cf.da_kwargs = {
        'do_elastic_deform': dim == 2,
        'alpha': (0., 1500.),
        'sigma': (30., 50.),
        'do_rotation': True,
        'angle_x': (0., 2 * np.pi) if dim == 2 else (0, 0.0),
        'angle_y': (0., 0) if dim == 2 else (0, 0.0),
        'angle_z': (0., 0) if dim == 2 else (0., 2 * np.pi),
        'do_scale': True,
        'scale': (0.8, 1.1),
        'random_crop': False,
        'rand_crop_dist': (cf.patch_size[0] / 2. - 3, cf.patch_size[1] / 2. - 3),
        'border_mode_data': 'constant',
        'border_cval_data': 0,
        'order_data': 1,
    }
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
    # evaluator (experiments/{lidc_exp,toy_exp,pet_ct_tnm_classification}/configs.py, default_configs.py); cf.fold is the cross-validation
    # fold being run (the reference's exec.py sets it per fold)
    cf.report_score_level = ['patient', 'rois']
    cf.patient_class_of_interest = 2
    cf.ap_match_ious = [0.1]
    cf.min_det_thresh = 0.1
    cf.model_selection_criteria = ['benign_ap', 'malignant_ap'] if exp == 'toy_exp' else ['malignant_ap', 'benign_ap']
    cf.per_patient_ap = False
    cf.scan_det_thresh = False
    cf.plot_prediction_histograms = True
    cf.plot_stat_curves = False
    cf.fold = 0
    cf.n_cv_splits = 5
    if exp == PETCT:
        cf.patient_class_of_interest = 1
        cf.model_selection_criteria = ['foreground_ap']
        # experiments/pet_ct_tnm_classification/configs.py: channels [0, 1], add_mrcnn_configs with one foreground class; its da_kwargs
        # equal the lidc values above for both dims
        cf.n_channels = 2
        cf.pre_crop_size = [300, 300] if dim == 2 else [280, 280, 48]
        cf.head_classes = 2
        cf.num_seg_classes = 2
        cf.class_specific_seg_flag = False
        cf.class_dict = {1: 'foreground'}
        cf.num_epochs = 100
        cf.learning_rate = [1e-4] * 50 + [5 * 1e-5] * 25 + [1e-5] * 25
        cf.return_masks_in_test = False
        cf.n_plot_rpn_props = 5 if dim == 2 else 30
    # data loader (data_loader.py; experiments/*/configs.py and default_configs.py, outside server_env).  The dataset paths and cf.exp_dir
    # are the user's to set.
    cf.experiment = exp
    if not hasattr(cf, 'pre_crop_size'):
        if exp == 'lidc_exp':
            cf.pre_crop_size = [300, 300] if dim == 2 else [156, 156, 96]
        elif dim == 2:
            cf.pre_crop_size = [320, 320]
    cf.seed = 0
    cf.server_env = False
    cf.input_df_name = 'info_df.pickle'
    cf.pp_data_path = cf.pp_test_data_path = cf.exp_dir = None
    cf.created_fold_id_pickle = False
    cf.hold_out_test_set = exp != 'lidc_exp'
    cf.select_prototype_subset = 100 if exp == 'lidc_exp' else None
    cf.batch_sample_slack = 0.2
    cf.n_3D_context = None
    cf.merge_2D_to_3D_preds = exp != 'toy_exp'
    cf.val_mode = 'val_patient' if exp == 'toy_exp' else 'val_sampling'
    cf.max_val_patients = None if exp == 'toy_exp' else 50
    cf.num_val_batches = 10 if exp == PETCT else 50
    cf.max_test_patients = 'all'
    cf.n_workers = 8
    if exp == 'toy_exp':
        cf.n_train_val_data = 1500
    if exp == PETCT:
        # petct_preprocessing.py (experiments/pet_ct_tnm_classification/configs.py); the raw and output paths are the user's to set
        cf.root_dir = cf.raw_data_dir = cf.pp_dir = None
    if exp == 'lidc_exp':
        # preprocessing.py (experiments/lidc_exp/configs.py:31-34); the raw and output paths are the user's to set
        cf.root_dir = cf.raw_data_dir = cf.pp_dir = None
        cf.target_spacing = (0.7, 0.7, 1.25)
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


def synthetic_precrop_batch(cf, src_shape, batch_size=None, seed=0, empty=(0,)):
    """A pre-crop batch as the reference's BatchGenerator yields it, for the augmentation (augment.py): uniform-noise image [B, C, *src_shape],
    uint8 instance map [B, 1, *src_shape] with several cuboid instances per element, class_target [B] lists (class 0 or 1 per id) and pid.
    Elements in `empty` have no foreground.  Ids leave gaps (some ids are never painted), some cuboids touch the source border and some lie
    in the margin a center crop to cf.patch_size cuts through or removes."""
    rs = np.random.RandomState(seed)
    B = batch_size or cf.batch_size
    dim = cf.dim
    S = [int(s) for s in src_shape[:dim]]
    P = cf.patch_size[:dim]
    data = rs.rand(B, cf.n_channels, *S).astype(np.float32)
    seg = np.zeros((B, 1, *S), dtype=np.uint8)
    class_target = []
    for b in range(B):
        if b in empty:
            class_target.append([])
            continue
        n_ids = int(rs.randint(3, 7))
        for k in range(1, n_ids + 1):
            kind = rs.randint(0, 4)                # 0: skipped id, 1: touches the border, 2: in the crop margin, 3: inside the patch
            if kind == 0 and k < n_ids:
                continue
            size = [int(rs.randint(3, max(4, min(20, S[d] // 4)))) for d in range(dim)]
            lo = []
            for d in range(dim):
                margin = max(0, (S[d] - P[d]) // 2)
                if kind == 1:
                    lo.append(0 if rs.rand() < 0.5 else S[d] - size[d])
                elif kind == 2 and d == 0 and margin > 1:
                    lo.append(int(rs.randint(0, margin)))
                else:
                    lo.append(int(rs.randint(margin, max(margin + 1, S[d] - margin - size[d]))))
            seg[(b, 0) + tuple(slice(lo[d], lo[d] + size[d]) for d in range(dim))] = k
        class_target.append([int(rs.randint(0, 2)) for _ in range(n_ids)])
    return {'data': data, 'seg': seg, 'class_target': class_target, 'pid': ['synth_%d' % i for i in range(B)]}


def synthetic_petct_precrop_batch(cf, src_shape=None, batch_size=None, seed=0, empty=(0,)):
    """A pre-crop batch as pet_ct_tnm_classification's BatchGenerator yields it, for the augmentation with get_rois_from_seg_flag=True:
    float16 noise image [B, cf.n_channels, *src_shape] (default cf.pre_crop_size), binary uint8 lesion map [B, 1, *src_shape] with several
    ellipsoid blobs per element (some overlapping or touching, so that they merge into one component, some in the margin a center crop to
    cf.patch_size cuts through or removes), scalar class_target per element (0 with foreground, -1 without) and pid.  Elements in `empty`
    have no foreground."""
    rs = np.random.RandomState(seed)
    B = batch_size or cf.batch_size
    dim = cf.dim
    S = [int(s) for s in (src_shape or cf.pre_crop_size)[:dim]]
    P = cf.patch_size[:dim]
    data = rs.rand(B, cf.n_channels, *S).astype(np.float16)
    seg = np.zeros((B, 1, *S), dtype=np.uint8)
    for b in range(B):
        if b in empty:
            continue
        centres = []
        for k in range(int(rs.randint(3, 8))):
            radius = [float(rs.uniform(2, max(3, min(12, S[d] / 6)))) for d in range(dim)]
            kind = rs.randint(0, 3)                # 0: next to the previous blob (merging or touching), 1: in the crop margin, 2: anywhere
            if kind == 0 and centres:
                c = [centres[-1][d] + rs.choice([-1, 1]) * radius[d] * rs.uniform(0.5, 1.5) for d in range(dim)]
            elif kind == 1:
                c = [float(rs.uniform(0, max(1, (S[0] - P[0]) / 2)))] + [float(rs.uniform(0, S[d])) for d in range(1, dim)]
            else:
                c = [float(rs.uniform(0, S[d])) for d in range(dim)]
            centres.append(c)
            lo = [max(0, int(np.floor(c[d] - radius[d]))) for d in range(dim)]
            hi = [min(S[d], int(np.ceil(c[d] + radius[d])) + 1) for d in range(dim)]
            if any(h <= l for l, h in zip(lo, hi)):
                continue
            ax = np.ogrid[tuple(slice(l, h) for l, h in zip(lo, hi))]
            inside = sum(((ax[d] - c[d]) / radius[d]) ** 2 for d in range(dim)) <= 1
            seg[(b, 0) + tuple(slice(l, h) for l, h in zip(lo, hi))][inside] = 1
    class_target = [0 if seg[b].any() else -1 for b in range(B)]
    return {'data': data, 'seg': seg, 'class_target': class_target, 'pid': ['synth_%d' % i for i in range(B)]}
