"""ctypes binding of libmdt_b200.so (the C-ABI declared in include/mdt_b200.h).

There is no fallback: if the shared library is missing or a call fails, an exception is raised.  PyTorch is used only for device
memory and the current CUDA stream.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmdt_b200.so")

c_i64p = ctypes.POINTER(ctypes.c_int64)


class MdtError(RuntimeError):
    pass


class PetctGrid(ctypes.Structure):
    """mirror of struct mdt_petct_grid (include/mdt_b200.h): an ITK image geometry in (x, y, z) order"""
    _fields_ = [("size", ctypes.c_int * 3), ("origin", ctypes.c_double * 3), ("spacing", ctypes.c_double * 3), ("direction", ctypes.c_double * 9)]


class Conv3dDesc(ctypes.Structure):
    """mirror of struct mdt_conv3d_desc (include/mdt_b200.h)"""
    _fields_ = [(n, ctypes.c_int) for n in (
        "n", "d", "h", "w", "cin", "cout", "kd", "kh", "kw", "sd", "sh", "sw", "pd", "ph", "pw", "relu", "precision", "algo")]


_lib = None

_VP = ctypes.c_void_p
_I = ctypes.c_int
_F = ctypes.c_float
_D = ctypes.c_double
_SZ = ctypes.c_size_t
_I64 = ctypes.c_int64

# name -> (restype, argtypes); every symbol declared in include/mdt_b200.h must appear here (tests/test_abi.py checks both directions)
SIGNATURES = {
    "mdt_version": (_I, []),
    "mdt_error_string": (ctypes.c_char_p, [_I]),
    "mdt_launch_count": (ctypes.c_ulonglong, []),
    "mdt_nms_mask_3d": (_I, [_I, _VP, _VP, _F, _VP]),
    "mdt_nms_mask_2d": (_I, [_I, _VP, _VP, _F, _VP]),
    "mdt_nms_workspace_bytes": (_SZ, [_I]),
    "mdt_nms_3d": (_I, [_VP, _I, _F, _VP, _SZ, _VP, _VP, _VP]),
    "mdt_nms_2d": (_I, [_VP, _I, _F, _VP, _SZ, _VP, _VP, _VP]),
    "mdt_crop_and_resize_3d_forward": (_I, [_VP, c_i64p, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _VP, c_i64p, _VP]),
    "mdt_crop_and_resize_3d_backward": (_I, [_VP, c_i64p, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _I, _VP, c_i64p, _I, _I64, _VP]),
    "mdt_crop_and_resize_2d_forward": (_I, [_VP, c_i64p, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _F, _VP, c_i64p, _VP]),
    "mdt_crop_and_resize_2d_backward": (_I, [_VP, c_i64p, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP, c_i64p, _I, _I64, _VP]),
    "mdt_pyramid_roi_align_forward": (_I, [_I, ctypes.POINTER(_VP), c_i64p, ctypes.POINTER(_I), _I, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP, c_i64p, _VP]),
    "mdt_pyramid_roi_align_backward": (_I, [_I, _VP, c_i64p, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, ctypes.POINTER(_VP), c_i64p, ctypes.POINTER(_I), _I, _I,
                                            c_i64p, _VP]),
    "mdt_anchor_match_workspace_bytes": (_SZ, [_I]),
    "mdt_anchor_match": (_I, [_I, _VP, _I, _VP, _VP, _I, _D, _D, _VP, _SZ, _VP, _VP, _VP, _VP]),
    "mdt_anchor_delta_targets": (_I, [_I, _VP, _VP, _VP, _VP, _I, _I, ctypes.POINTER(_D), _VP, _VP]),
    "mdt_conv3d_workspace_bytes": (_SZ, [ctypes.POINTER(Conv3dDesc), _I]),
    "mdt_conv3d_fprop": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_conv3d_dgrad": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_conv3d_wgrad": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_conv3d_algo": (_I, [ctypes.POINTER(Conv3dDesc), _I]),
    "mdt_conv3d_variant": (_I, [ctypes.POINTER(Conv3dDesc), _I]),
    "mdt_conv3d_backward_fused": (_I, [ctypes.POINTER(Conv3dDesc), _I]),
    "mdt_conv3d_backward_workspace_bytes": (_SZ, [ctypes.POINTER(Conv3dDesc), _I]),
    "mdt_conv3d_backward": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_conv3d_split_bytes": (_SZ, [ctypes.POINTER(Conv3dDesc)]),
    "mdt_conv3d_split": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP]),
    "mdt_conv3d_fprop_presplit": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_conv3d_out_split_bytes": (_SZ, [ctypes.POINTER(Conv3dDesc)]),
    "mdt_conv3d_fprop_presplit_out": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_conv3d_fprop_out": (_I, [ctypes.POINTER(Conv3dDesc), _VP, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_upsample221_forward": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mdt_upsample221_backward": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mdt_upsample_linear2x_forward": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mdt_upsample_linear2x_backward": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mdt_maxpool3d_forward": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, ctypes.POINTER(_I), ctypes.POINTER(_I), ctypes.POINTER(_I), _VP]),
    "mdt_maxpool3d_backward": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, ctypes.POINTER(_I), ctypes.POINTER(_I), ctypes.POINTER(_I), _VP]),
    "mdt_upsample_nearest_forward": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "mdt_upsample_nearest_backward": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "mdt_seg_loss_workspace_bytes": (_SZ, [_I]),
    "mdt_seg_loss_forward": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _F, _F, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_seg_loss_backward": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _F, _F, _VP, _VP, _VP, _VP]),
    "mdt_seg_loss_weighted_forward": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _F, _F, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_seg_loss_weighted_backward": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _F, _F, _VP, _VP, _VP, _VP, _VP]),
    "mdt_seg_loss_sample_workspace_bytes": (_SZ, [_I, _I64, _I]),
    "mdt_seg_loss_sample_sums": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _VP, _VP, _SZ, _VP]),
    "mdt_seg_loss_weighted_sample_sums": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_seg_loss_from_sums": (_I, [_VP, _I, _I64, _I, _F, _F, _VP, _VP, _VP, _VP]),
    "mdt_seg_loss_backward_global": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _F, _F, _VP, _I64, _VP, _I, _VP, _VP]),
    "mdt_seg_loss_weighted_backward_global": (_I, [_VP, c_i64p, _VP, _I, _I64, _I, _F, _F, _VP, _VP, _I64, _VP, _I, _VP, _VP]),
    "mdt_exchange_fill": (_I, [_VP, _I64, _I, _VP]),
    "mdt_seg_components_workspace_bytes": (_SZ, [_I, _I, _I, _I, _I, _I, _I, _I]),
    "mdt_seg_components": (_I, [_VP, c_i64p, _I, _I, _I, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_shem_workspace_bytes": (_SZ, [_I, _I]),
    "mdt_shem_class_loss_forward": (_I, [_VP, _VP, _I, _I, _VP, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_shem_class_loss_backward": (_I, [_VP, _I, _I, _VP, _VP, _VP, _I, _VP, _VP, _VP]),
    "mdt_wbc_workspace_bytes": (_SZ, [_I, _I]),
    "mdt_wbc": (_I, [_VP, _VP, _VP, _I, _I, _I, _D, _D, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_nms_2to3d_workspace_bytes": (_SZ, [_I, _I]),
    "mdt_nms_2to3d": (_I, [_VP, _VP, _I, _D, _I, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_norm_workspace_bytes": (_SZ, [_I, _I64, _I, _I]),
    "mdt_norm_stats": (_I, [_VP, _I, _I64, _I, _I, _F, _F, _VP, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_norm_eval_stats": (_I, [_VP, _VP, _I, _F, _VP, _VP, _VP]),
    "mdt_norm_apply": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I64, _I, _I, _I, _F, _VP, _VP]),
    "mdt_norm_backward": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I64, _I, _I, _I, _F, _I, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_norm_sample_workspace_bytes": (_SZ, [_I, _I64, _I]),
    "mdt_norm_sample_sums": (_I, [_VP, _I, _I64, _I, _VP, _VP, _SZ, _VP]),
    "mdt_norm_stats_from_sums": (_I, [_VP, _I, _I64, _I, _F, _F, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mdt_norm_backward_sample_sums": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I64, _I, _I, _F, _VP, _VP, _SZ, _VP]),
    "mdt_norm_backward_from_sums": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I64, _I, _I, _F, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_act_forward": (_I, [_VP, _I64, _I, _F, _VP, _VP]),
    "mdt_act_backward": (_I, [_VP, _VP, _I64, _I, _F, _VP, _VP]),
    "mdt_augment_gaussian_workspace_bytes": (_SZ, [_I, _I, ctypes.POINTER(_I)]),
    "mdt_augment_gaussian": (_I, [_I, _VP, _I, ctypes.POINTER(_I), ctypes.POINTER(_D), ctypes.POINTER(_D), _VP, _VP, _SZ, _VP]),
    "mdt_augment_spatial_workspace_bytes": (_SZ, [_I, _I, _I, ctypes.POINTER(_I)]),
    "mdt_augment_spatial": (_I, [_I, _VP, _VP, _I, _I, ctypes.POINTER(_I), ctypes.POINTER(_I), _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_augment_seg_to_boxes": (_I, [_I, _VP, _I, ctypes.POINTER(_I), _VP, _I, _VP, _VP, _VP, _VP]),
    "mdt_seg_rois_workspace_bytes": (_SZ, [_I, _I, ctypes.POINTER(_I)]),
    "mdt_seg_rois": (_I, [_I, _VP, _I, ctypes.POINTER(_I), _VP, _I, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_seg_rois_masks": (_I, [_I, _VP, _I, ctypes.POINTER(_I), _VP, _I, _VP, _VP]),
    "mdt_eval_match_workspace_bytes": (_SZ, [_I, _I, _I, _I]),
    "mdt_eval_match": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _I, _VP, _I, _I, _I, _VP, _I, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_eval_roi_ap_workspace_bytes": (_SZ, [_I, _I]),
    "mdt_eval_roi_ap": (_I, [_VP, _VP, _VP, _I, _I, _VP, _I, _VP, _I, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_eval_patient_workspace_bytes": (_SZ, [_I, _I]),
    "mdt_eval_patient": (_I, [_VP, _VP, _VP, _I, _I, _VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_eval_bootstrap_roi_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mdt_eval_bootstrap_roi": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP, _I, _D, _VP, _I, _VP, _I, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_eval_bootstrap_patient_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mdt_eval_bootstrap_patient": (_I, [_VP, _VP, _VP, _VP, _I, _I, _VP, _VP, _I, _I, _I, _VP, _I, _VP, _VP, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_unmold_masks": (_I, [_I, _VP, _I, _VP, c_i64p, _I, ctypes.POINTER(_I), _I, ctypes.POINTER(_I), _VP, _VP, _VP]),
    "mdt_loader_fg_index_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mdt_loader_fg_index": (_I, [_VP, _I, _I, _I, _VP, _VP, _I, _VP, _SZ, _VP]),
    "mdt_loader_gather": (_I, [_I, _VP, _VP, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _I, _VP, _VP]),
    "mdt_pp_resample_workspace_bytes": (_SZ, [ctypes.POINTER(_I), ctypes.POINTER(_I)]),
    "mdt_pp_resample": (_I, [_I, _VP, ctypes.POINTER(_I), ctypes.POINTER(_I), _VP, _VP, _SZ, _VP]),
    "mdt_pp_normalize_workspace_bytes": (_SZ, [_I64]),
    "mdt_pp_normalize": (_I, [_VP, _I64, _VP, _VP, _SZ, _VP]),
    "mdt_pp_vote_add": (_I, [_VP, _VP, _I64, _I, _VP]),
    "mdt_pp_vote_label": (_I, [_VP, _I64, _I, _I, _VP, _VP, _VP]),
    "mdt_pp_label_summary": (_I, [_VP, _I, _I64, _VP, _VP, _VP]),
    "mdt_petct_resample": (_I, [_I, _VP, ctypes.POINTER(PetctGrid), _I, _VP, ctypes.POINTER(PetctGrid), _VP]),
    "mdt_petct_seg_merge": (_I, [_I, _VP, _I, _I, _I, _I, c_i64p, ctypes.POINTER(ctypes.c_ubyte), _VP, _VP]),
    "mdt_petct_body_components_capacity": (_I64, [_I, _I, _I]),
    "mdt_petct_body_components_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mdt_petct_body_components": (_I, [_I, _VP, _I, _I, _I, _VP, _VP, _VP, _I64, _VP, _SZ, _VP]),
    "mdt_petct_zcrop_criterion": (_I, [_VP, _VP, _I, _I, _I, _I64, _I, _D, _VP, _VP]),
    "mdt_petct_normalize_workspace_bytes": (_SZ, [_I64]),
    "mdt_petct_normalize": (_I, [_VP, _VP, _I64, _VP, _VP, _VP, _SZ, _VP]),
    "mdt_toy_images": (_I, [_VP, _I, _I, _I, _I, _I, _VP, _VP, _VP]),
    "mdt_render_panel_range": (_I, [_VP, _I, _VP, _VP]),
    "mdt_render_panels": (_I, [_VP, _I, _VP, _VP, _I, _VP, _I, _I, _VP]),
    "mdt_render_prims": (_I, [_VP, _I, _VP, _I, _I, _VP]),
}


def load():
    """Load libmdt_b200.so once; raises MdtError if it has not been built (run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MdtError("libmdt_b200.so not found at %s - build it with `make -C medicaldetectiontoolkit_b200/csrc` "
                       "(there is no CPU or PyTorch fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header / library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code):
    if code != 0:
        raise MdtError("libmdt_b200: %s (code %d)" % (load().mdt_error_string(code).decode(), code))


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def i64arr(vals):
    return (ctypes.c_int64 * len(vals))(*[int(v) for v in vals])


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise MdtError("libmdt_b200 ops take CUDA tensors only (no CPU fallback); got a %s tensor" % t.device)
