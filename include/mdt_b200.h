/*
 * mdt_b200.h — C-ABI of libmdt_b200.so: the H100 (sm_90a) drop-in for the native ops of
 * MIC-DKFZ/medicaldetectiontoolkit's detection hot path.
 *
 * Conventions (all entry points):
 *   - plain pointers + sizes, no framework types; every pointer is a DEVICE pointer unless the
 *     parameter name ends in _host;
 *   - the caller owns all memory including scratch ("workspace"); query sizes with *_workspace_bytes;
 *   - work is enqueued on the caller's `stream` (a cudaStream_t passed as void*); no host sync inside;
 *   - return value: 0 = success, <0 = MDT_E* argument error, >0 = cudaError_t of the failed launch.
 *     Nothing ever calls exit() (the reference's launchers do: roi_align_3D/.../crop_and_resize_kernel.cu:326-331).
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference root).
 */
#ifndef MDT_B200_H
#define MDT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDT_OK 0
#define MDT_EINVAL (-1)     /* bad argument (null pointer, negative size, unsupported shape) */
#define MDT_EWORKSPACE (-2) /* workspace too small */
#define MDT_EUNSUPPORTED (-3)
#define MDT_EDRIVER (-4)    /* driver entry point (tensor-map encode) unavailable or failed */

int mdt_version(void);
/* human-readable text for a return code of any entry point */
const char *mdt_error_string(int code);

/* ------------------------------------------------------------------ NMS ------------------------------------------------------------------
 * replaces: cuda_functions/nms_3D/src/cuda/nms_kernel.h:11-12  `void _nms(int boxes_num, float* boxes_dev, unsigned long long* mask_dev, float thresh)`
 *           cuda_functions/nms_3D/src/nms_cuda.h:1             `int gpu_nms(THLongTensor* keep, THLongTensor* num_out, THCudaTensor* boxes, float thresh)`
 *           (2D twins under cuda_functions/nms_2D/)
 * boxes are sorted by descending score: 3D rows = (y1,x1,y2,x2,z1,z2,score) [N,7] f32, 2D rows = (y1,x1,y2,x2,score) [N,5] f32, contiguous.
 * IoU uses +1 extents and the strict `>` of nms_kernel.cu:16-28,71.
 */

/* bitmask only — same contract as the reference `_nms` plus stream/status; mask is [N, ceil(N/64)] u64, fully written */
int mdt_nms_mask_3d(int boxes_num, const float *boxes_dev, unsigned long long *mask_dev, float nms_overlap_thresh, void *stream);
int mdt_nms_mask_2d(int boxes_num, const float *boxes_dev, unsigned long long *mask_dev, float nms_overlap_thresh, void *stream);

/* fused: bitmask + ON-DEVICE greedy reduction (replaces the D2H copy + host loop of nms_cuda.c:33-61).
 * keep_out [N] int64: first *num_out entries are the kept row indices (into the sorted input), ascending; num_out [1] int32 (device).
 * workspace: the upper-triangular mask [N][ceil(N/64)] u64 followed by the reduction's suppression bitmap and control block; the
 * reduction is a cooperative launch (<= one CTA per SM) that the call zero-initialises itself - the caller only provides the bytes. */
size_t mdt_nms_workspace_bytes(int boxes_num);
int mdt_nms_3d(const float *boxes_dev, int boxes_num, float nms_overlap_thresh, void *workspace, size_t workspace_bytes,
               int64_t *keep_out, int *num_out, void *stream);
int mdt_nms_2d(const float *boxes_dev, int boxes_num, float nms_overlap_thresh, void *workspace, size_t workspace_bytes,
               int64_t *keep_out, int *num_out, void *stream);

/* --------------------------------------------------------------- RoIAlign ----------------------------------------------------------------
 * replaces: cuda_functions/roi_align_3D/roi_align/src/cuda/crop_and_resize_kernel.h:8-18 (CropAndResizeLaucher / CropAndResizeBackpropImageLaucher)
 *           and the 2D twins. Same argument order; added: element strides of the image (so channels-last maps need no copy) and int status.
 * image  logical [batch, depth(C), H, W, Z] f32 with element strides img_strides[5] (2D: [batch, C, H, W], img_strides[4])
 * boxes  [num_boxes, 6] f32 normalised (y1,x1,y2,x2,z1,z2)   (2D: [num_boxes,4])
 * box_ind[num_boxes] int32 in [0,batch); out-of-range => that crop stays zero (crop_and_resize_kernel.cu:43-47 + crop_and_resize_gpu.c:27)
 * crops  logical [num_boxes, C, ch, cw, cz] f32 with element strides crop_strides[5]; fully written (zeros for bad box_ind).
 * extrapolation_value is accepted and ignored, as in the reference GPU kernel.
 */
int mdt_crop_and_resize_3d_forward(const float *image, const int64_t *img_strides_host, const float *boxes, const int *box_ind, int num_boxes,
                                   int batch, int image_height, int image_width, int image_zdepth, int crop_height, int crop_width,
                                   int crop_zdepth, int depth, float extrapolation_value, float *crops, const int64_t *crop_strides_host,
                                   void *stream);
/* backward: a gather in a fixed order (csrc/roi_align.cu), so two calls with the same arguments give the same bits.  Every logical element of
 * grads_image is written once: zero_init=1 gives the sum of the RoI terms, zero_init=0 adds them to the element's prior content; elements between
 * strided rows are not touched.  image_numel (> 0 with zero_init=1) is the caller's extent of grads_image, as before. */
int mdt_crop_and_resize_3d_backward(const float *grads, const int64_t *grad_strides_host, const float *boxes, const int *box_ind, int num_boxes,
                                    int batch, int image_height, int image_width, int image_zdepth, int crop_height, int crop_width,
                                    int crop_zdepth, int depth, float *grads_image, const int64_t *img_strides_host, int zero_init,
                                    int64_t image_numel, void *stream);
int mdt_crop_and_resize_2d_forward(const float *image, const int64_t *img_strides_host, const float *boxes, const int *box_ind, int num_boxes,
                                   int batch, int image_height, int image_width, int crop_height, int crop_width, int depth,
                                   float extrapolation_value, float *crops, const int64_t *crop_strides_host, void *stream);
int mdt_crop_and_resize_2d_backward(const float *grads, const int64_t *grad_strides_host, const float *boxes, const int *box_ind, int num_boxes,
                                    int batch, int image_height, int image_width, int crop_height, int crop_width, int depth,
                                    float *grads_image, const int64_t *img_strides_host, int zero_init, int64_t image_numel, void *stream);

/* pyramid RoIAlign: ONE launch over all FPN levels.  replaces: models/mrcnn.py:373-457 pyramid_roi_align's per-level loop (boolean-mask gather,
 * up to 4 CropAndResize calls, concat, un-permute through a sort).  roi_level[n] in [0, nlevels) selects the map of RoI n (the reference's
 * round(4 + log2(sqrt(h*w))) rule is evaluated by the caller); every crop row is written exactly once, bad box_ind rows are zeros.
 * images / grad_images: HOST arrays of nlevels device pointers (channels-last maps, C % 4 == 0); image_strides: nlevels x 5 int64 element strides
 * (b, c, y, x, z); image_dims: nlevels x 3 (H, W, Z).  Returns MDT_EUNSUPPORTED for layouts outside the vector kernel (caller then loops over
 * levels with mdt_crop_and_resize_*).  dim = 2 or 3 (2: crop_zdepth and the Z entries are ignored).  The backward is the single-map entry
 * point's gather, each level's map receiving its own RoIs (image_numel: nlevels extents, > 0 with zero_init=1). */
int mdt_pyramid_roi_align_forward(int dim, const float *const *images, const int64_t *image_strides, const int *image_dims, int nlevels, const float *boxes,
                                  const int *box_ind, const int *roi_level, int num_boxes, int batch, int crop_height, int crop_width, int crop_zdepth,
                                  int depth, float *crops, const int64_t *crop_strides, void *stream);
int mdt_pyramid_roi_align_backward(int dim, const float *grads, const int64_t *grad_strides, const float *boxes, const int *box_ind, const int *roi_level,
                                   int num_boxes, int batch, int crop_height, int crop_width, int crop_zdepth, int depth, float *const *grad_images,
                                   const int64_t *image_strides, const int *image_dims, int nlevels, int zero_init, const int64_t *image_numel, void *stream);

/* ------------------------------------------------------------ anchor <-> GT matching --------------------------------------------------------
 * replaces: utils/model_utils.py:505-619 gt_anchor_matching (+ compute_overlaps :83-110, compute_iou_{2D,3D} :35-79), which runs in numpy f64 on the host.
 * anchors [A, 2*dim] f64, gt_boxes [G, 2*dim] f64, gt_class_ids [G] int32 (NULL => all 1, the RPN case of mrcnn.py:894).
 * Outputs (device):
 *   matches   [A] int32   : -1 negative / 0 neutral / class id positive — state BEFORE the random sub-sampling of model_utils.py:566-571
 *   iou_argmax[A] int32   : row argmax (first index on ties, numpy semantics) — needed by the caller for delta targets
 *   n_pos     [1] int32   : number of positive anchors
 * neg_iou_thresh is 0.01 (3D) / 0.1 (2D) in the reference (:549-552); pos_iou_thresh = cf.anchor_matching_iou.
 * workspace: mdt_anchor_match_workspace_bytes(G).
 */
size_t mdt_anchor_match_workspace_bytes(int num_gt);
int mdt_anchor_match(int dim, const double *anchors, int num_anchors, const double *gt_boxes, const int *gt_class_ids, int num_gt,
                     double neg_iou_thresh, double pos_iou_thresh, void *workspace, size_t workspace_bytes, int *matches, int *iou_argmax,
                     int *n_pos, void *stream);
/* delta targets for up to max_targets positive anchors in ascending anchor order (model_utils.py:573-617): out [max_targets, 2*dim] f64, zero padded.
 * pos_ids [n_pos] int32 ascending anchor indices (after any sub-sampling done by the caller). std_dev [2*dim] f64 (host). */
int mdt_anchor_delta_targets(int dim, const double *anchors, const double *gt_boxes, const int *iou_argmax, const int *pos_ids, int n_pos,
                             int max_targets, const double *std_dev_host, double *targets_out, void *stream);

/* ------------------------------------------------------------------ conv3d ----------------------------------------------------------------
 * replaces: the nn.Conv3d (+bias, +ReLU) built by utils/model_utils.py:739-781 NDConvGenerator and consumed by models/backbone.py:27-206.
 * Layout: activations NDHWC ("channels_last_3d"): x [N, D, H, W, C] f32 contiguous, where (D,H,W) are the reference's (y,x,z) axes.
 *         weights in the reference's parameter layout [Cout, Cin, kd, kh, kw] f32 contiguous (state-dict compatible).
 * Descriptor struct keeps the signature stable across kernels.
 */
typedef struct mdt_conv3d_desc {
    int n, d, h, w;          /* input batch and spatial extent */
    int cin, cout;
    int kd, kh, kw;
    int sd, sh, sw;          /* strides */
    int pd, ph, pw;          /* zero padding */
    int relu;                /* fuse ReLU into the fprop epilogue */
    int precision;           /* 0 = fp32-faithful (3-pass split-bf16 on the tensor cores, or fp32 SIMT); 1 = single-pass bf16 (throughput mode) */
    int algo;                /* 0 = auto, 1 = force SIMT direct kernels, 2 = force tensor-core (wgmma) implicit GEMM, 4 = force pointwise streaming (error if unsupported) */
} mdt_conv3d_desc;

size_t mdt_conv3d_workspace_bytes(const mdt_conv3d_desc *desc_host, int pass /*0 fprop,1 dgrad,2 wgrad*/);
/* y = relu?(conv(x, w) + bias); bias may be NULL; residual (same shape as y, may be NULL) is added before the ReLU.
 * The fused ReLU keeps NaN, as torch.relu does; the ReLU mask of mdt_conv3d_backward zeroes dy where y_relu <= 0 and passes it where
 * y_relu is NaN, as aten::threshold_backward does. */
int mdt_conv3d_fprop(const mdt_conv3d_desc *desc_host, const float *x, const float *w, const float *bias, const float *residual, float *y,
                     void *workspace, size_t workspace_bytes, void *stream);
/* dx = conv_transpose(dy, w) */
int mdt_conv3d_dgrad(const mdt_conv3d_desc *desc_host, const float *dy, const float *w, float *dx, void *workspace, size_t workspace_bytes,
                     void *stream);
/* dw = x (*) dy ; db = sum(dy) (db may be NULL) */
int mdt_conv3d_wgrad(const mdt_conv3d_desc *desc_host, const float *x, const float *dy, float *dw, float *db, void *workspace,
                     size_t workspace_bytes, void *stream);
/* Fused backward of one conv layer (tensor-core path): ONE streaming pass over dy yields the split-bf16 operand shared by dgrad and wgrad, applies
 * the ReLU mask of a fused-ReLU conv (y_relu = its forward output, NULL = no mask; replaces aten::threshold_backward of the reference graph),
 * accumulates db, and optionally writes the masked fp32 gradient (dy_masked_out, needed as the gradient of a fused residual input; a copy of
 * dy when y_relu is NULL).  The same contract holds on the pointwise path (1x1x1 convs, fp32 streaming dgrad + wgrad).
 * dx may be NULL (first layer).  mdt_conv3d_backward_fused() tells whether this path applies; otherwise use dgrad + wgrad.
 * x_split (optional, else NULL and x is split internally): the canonical split form of x produced by mdt_conv3d_split. */
int mdt_conv3d_backward_fused(const mdt_conv3d_desc *desc_host, int need_dx);
size_t mdt_conv3d_backward_workspace_bytes(const mdt_conv3d_desc *desc_host, int need_dx);
int mdt_conv3d_backward(const mdt_conv3d_desc *desc_host, const float *x, const void *x_split, const float *dy, const float *y_relu,
                        const float *w, float *dx, float *dw, float *db, float *dy_masked_out, void *workspace, size_t workspace_bytes,
                        void *stream);
/* Canonical split form of an activation tensor (two bf16 planes, channels padded, W-line interleaved): it depends on the tensor alone, so ONE
 * split serves every conv that reads the tensor (sibling layers, fprop and the later weight gradient).  mdt_conv3d_split_bytes gives the buffer
 * size for the INPUT x of `desc`; mdt_conv3d_fprop_presplit is mdt_conv3d_fprop on such a buffer (tensor-core path only, else MDT_EUNSUPPORTED). */
size_t mdt_conv3d_split_bytes(const mdt_conv3d_desc *desc_host);
int mdt_conv3d_split(const mdt_conv3d_desc *desc_host, const float *x, void *x_split, void *stream);
int mdt_conv3d_fprop_presplit(const mdt_conv3d_desc *desc_host, const void *x_split, const float *w, const float *bias, const float *residual,
                              float *y, void *workspace, size_t workspace_bytes, void *stream);
/* mdt_conv3d_fprop_presplit that ALSO emits the result y in canonical split form (mdt_conv3d_out_split_bytes bytes; layout of mdt_conv3d_split
 * applied to y, padding channels zero) from the conv epilogue: the consumer conv then needs no split pass over y (tensor-core path only). */
size_t mdt_conv3d_out_split_bytes(const mdt_conv3d_desc *desc_host);
int mdt_conv3d_fprop_presplit_out(const mdt_conv3d_desc *desc_host, const void *x_split, const float *w, const float *bias, const float *residual,
                                  float *y, void *y_split, void *workspace, size_t workspace_bytes, void *stream);
/* fp32-input fprop that also emits the split planes of y (as mdt_conv3d_fprop_presplit_out does for a pre-split input): pointwise path only
 * (mdt_conv3d_algo == 4), else MDT_EUNSUPPORTED.  Used where a 1x1x1 conv feeds a tensor-core conv (ResBlock conv1 -> conv2, P0_conv1 -> P0_conv2). */
int mdt_conv3d_fprop_out(const mdt_conv3d_desc *desc_host, const float *x, const float *w, const float *bias, const float *residual, float *y,
                         void *y_split, void *workspace, size_t workspace_bytes, void *stream);
/* which algorithm `auto` resolves to for this descriptor/pass: 1 SIMT, 2 tensor-core implicit GEMM, 4 pointwise fp32 streaming (1x1x1, stride 1, no padding,
 * cin * cout <= 2592 under `auto` (the HBM-bound layers), <= 6144 when forced with algo = 4: HBM-bound layers, csrc/conv3d_pw.cu) */
int mdt_conv3d_algo(const mdt_conv3d_desc *desc_host, int pass);
/* which kernel family runs this descriptor/pass: 1 fp32 SIMT / direct stem, 2 wgmma halo-window implicit GEMM (conv3d_tc.cu, wgrad:
 * conv3d_tc_wgrad.cu), 4 pointwise fp32 streaming (conv3d_pw.cu); 0 = unsupported */
int mdt_conv3d_variant(const mdt_conv3d_desc *desc_host, int pass);
/* ------------------------------------------------------------- decoder up-sampling -----------------------------------------------------------
 * replaces: F.interpolate(x, scale_factor=(2,2,1), mode='trilinear', align_corners=False) of models/backbone.py:209-218 (P2/P1_upsample), NDHWC.
 * x [n, d, h, w, c] -> y [n, 2d, 2h, w, c]; c % 4 == 0 and every pointer 16-byte aligned (float4 accesses), else MDT_EINVAL; backward is the exact
 * adjoint, written as a gather (no atomics, no zero fill). */
int mdt_upsample221_forward(const float *x, float *y, int n, int d, int h, int w, int c, void *stream);
int mdt_upsample221_backward(const float *gy, float *gx, int n, int d, int h, int w, int c, void *stream);
/* The same (2,2,1) map and gather adjoint for any c >= 1 and fp32 pointers aligned to 4 bytes (else MDT_EINVAL), accessing V = 4, 2 or 1
 * channels at a time as the pooling kernels below do.  Also replaces F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False) of
 * the 2D decoder: an NHWC map is passed with w = 1.  Each element's arithmetic and its order of the 16 gather terms do not depend on V: the
 * result equals mdt_upsample221_* bit for bit where both accept the arguments, and the backward is bit-reproducible. */
int mdt_upsample_linear2x_forward(const float *x, float *y, int n, int d, int h, int w, int c, void *stream);
int mdt_upsample_linear2x_backward(const float *gy, float *gx, int n, int d, int h, int w, int c, void *stream);

/* ------------------------------------------------------------- pooling / nearest up-sampling -------------------------------------------------
 * replaces: nn.MaxPool3d(kernel_size=3, stride=(2,2,1), padding=1) / nn.MaxPool2d(3, 2, 1) of models/backbone.py:63-64 (applied at :129) and its
 * autograd backward.  NDHWC maps (2D: d = 1, kernel {1,3,3}).  x [n,d,h,w,c] -> y [n,od,oh,ow,c] with o = (i + 2p - k) / s + 1 (floor mode);
 * argmax [n,od,oh,ow,c] holds the winning window offset ((a*kh + b)*kw + e) per element, ATen's update rule (first maximum, NaN propagates).
 * Backward is a gather over the windows containing an input voxel: no atomics, gx fully written.
 * Pooling and nearest up-sampling access V = 4, 2 or 1 channels at a time: the widest V that divides c and to whose 4V-byte boundary every fp32
 * pointer is aligned (a view with a storage offset may start anywhere); fp32 pointers that are not 4-byte aligned return MDT_EINVAL. */
int mdt_maxpool3d_forward(const float *x, float *y, unsigned char *argmax, int n, int d, int h, int w, int c, const int *kernel3, const int *stride3,
                          const int *pad3, void *stream);
int mdt_maxpool3d_backward(const float *gy, const unsigned char *argmax, float *gx, int n, int d, int h, int w, int c, const int *kernel3,
                           const int *stride3, const int *pad3, void *stream);
/* replaces: F.interpolate(x, scale_factor=2) (mode 'nearest') of the FPN top-down path, models/backbone.py:147-153.  x [n,d,h,w,c] ->
 * y [n,d*fd,h*fh,w*fw,c], factors 1 or 2 per axis; backward sums the children of each input voxel (gather, gx fully written). */
int mdt_upsample_nearest_forward(const float *x, float *y, int n, int d, int h, int w, int c, int fd, int fh, int fw, void *stream);
int mdt_upsample_nearest_backward(const float *gy, float *gx, int n, int d, int h, int w, int c, int fd, int fh, int fw, void *stream);

/* ------------------------------------------------------------- loss-side kernels (csrc/loss_ops.cu) ------------------------------------------
 * Segmentation loss.  replaces: F.softmax(seg_logits, 1) + get_one_hot_encoding + batch_dice (utils/model_utils.py:785-799, 833-858) and
 * F.cross_entropy(seg_logits, seg[:, 0]) of models/retina_unet.py:395,446-448 (same calls in models/mrcnn.py is n/a; ufrcnn.py uses them too).
 * logits[b, c, v] = logits + b*strides3[0] + c*strides3[1] + v*strides3[2] (elements; NCDHW: {C*V, V, 1}, channels-last: {V*C, 1, C});
 * target uint8 [n, voxels]; n_classes <= 8.  sums (device, 3*n_classes + 1 doubles) = per-class intersect, sum p, sum y, then sum(-log p_t) —
 * saved for the backward; out2 (device) = {dice score (mean over foreground classes, batch pseudo-volume), mean cross-entropy}.
 * Deterministic (fixed-order fp64 reduction).  backward: grad_out2 (device) = {dL/d dice_score, dL/d ce}; grad_logits has logits' strides. */
size_t mdt_seg_loss_workspace_bytes(int n_classes);
int mdt_seg_loss_forward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                         float false_positive_weight, float smooth, double *sums, float *out2, void *ws, size_t ws_bytes, void *stream);
int mdt_seg_loss_backward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                          float false_positive_weight, float smooth, const double *sums, const float *grad_out2, float *grad_logits, void *stream);
/* Class-weighted variant.  replaces: 1 - batch_dice(F.softmax(seg_logits), one_hot, false_positive_weight=fp_dice_weight) and
 * F.cross_entropy(seg_logits, seg, weight=wce_weights) of models/detection_unet.py:124-130.  class_weights (device, n_classes floats) != NULL;
 * out2[1] = sum_v w[t_v] (-log p_{t_v}) / sum_v w[t_v]; sums[3C] holds the weighted numerator.  Same workspace, dice term and fixed-order fp64
 * reductions as mdt_seg_loss_forward; with all weights 1 the results are bit-identical to the unweighted entry points. */
int mdt_seg_loss_weighted_forward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                  float false_positive_weight, float smooth, const float *class_weights, double *sums, float *out2, void *ws,
                                  size_t ws_bytes, void *stream);
int mdt_seg_loss_weighted_backward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                   float false_positive_weight, float smooth, const float *class_weights, const double *sums, const float *grad_out2,
                                   float *grad_logits, void *stream);
/* The seg loss of a batch split across ranks.  mdt_seg_loss_sample_sums (+ _weighted): rows (device, [n][3*n_classes + 1] doubles) = the sums
 * layout above for each sample alone; the grid is (sample, chunk) with a chunk count that depends on (voxels, n_classes) only and every sum is
 * fp64 in a fixed order, so a sample's row is bit-identical in a batch of any size.  Workspace: mdt_seg_loss_sample_workspace_bytes (0 =
 * unsupported arguments).  mdt_seg_loss_from_sums: rows [n_total][3*n_classes + 1] (all ranks' rows, rank-major) added in row order -> sums and
 * out2 as mdt_seg_loss_forward; the unweighted CE denominator is n_total * voxels, the weighted one sum_c w[c] tsum_c (class_weights NULL =
 * unweighted).  mdt_seg_loss_backward_global (+ _weighted): mdt_seg_loss_backward over this rank's n samples with the global sums and the
 * unweighted CE denominator total_voxels (>= n * voxels); grad_out2 holds n_ranks >= 1 pairs {dL/d dice_score, dL/d ce} (every rank's, in
 * rank order), added in fp64 in that order.
 * mdt_exchange_fill: count elements of buf set to -0.0 (f64 = 1: doubles, 0: floats), the fill of an exchange buffer whose slots each rank
 * writes before an all_reduce(SUM): v + (-0.0) = v for every v, so every slot arrives with its bits. */
size_t mdt_seg_loss_sample_workspace_bytes(int n, long long voxels, int n_classes);
int mdt_seg_loss_sample_sums(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                             double *rows, void *ws, size_t ws_bytes, void *stream);
int mdt_seg_loss_weighted_sample_sums(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels,
                                      int n_classes, const float *class_weights, double *rows, void *ws, size_t ws_bytes, void *stream);
int mdt_seg_loss_from_sums(const double *rows, int n_total, long long voxels, int n_classes, float false_positive_weight, float smooth,
                           const float *class_weights, double *sums, float *out2, void *stream);
int mdt_seg_loss_backward_global(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                 float false_positive_weight, float smooth, const double *sums, long long total_voxels, const float *grad_out2,
                                 int n_ranks, float *grad_logits, void *stream);
int mdt_seg_loss_weighted_backward_global(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels,
                                          int n_classes, float false_positive_weight, float smooth, const float *class_weights, const double *sums,
                                          long long total_voxels, const float *grad_out2, int n_ranks, float *grad_logits, void *stream);
int mdt_exchange_fill(void *buf, long long count, int f64, void *stream);

/* ------------------------------------------------------------- segmentation connected components (csrc/seg_components.cu) ------------------
 * replaces: softmax + D2H copy + per-class argmax mask + get_coords (scipy.ndimage.label, np.unique, argsort, one full-volume mask per kept
 * component) + the per-component max/median score loop of models/detection_unet.py:58-85,170-213.
 * logits [n, S, y, x, z] fp32 with element strides3 = {batch, class, voxel} (voxel index in (y, x, z) C order; 2D: z = 1, dim = 2).
 * S = n_seg_classes <= 8; n_fg_classes = C_fg = len(class_dict) (classes 1..C_fg are labelled; a class without a channel has no component);
 * 1 <= k <= 128 components kept per (element, class); n*y*x*z < 2^31 and n*C_fg*k < 2^31; median != 0 scores by the exact median instead of the max.
 * Outputs (device): seg_pred uint8 [n, y, x, z] = argmax of the softmax (first index on ties); comp_label int32 [n, y, x, z] (optional, NULL to
 * skip) = dense component id in scipy's label order, -1 for background; boxes int32 [n, C_fg, k, 2*dim] = (y1, x1, y2, x2, (z1, z2)) padded and
 * clipped as get_coords does; scores f32 [n, C_fg, k]; n_kept int32 [n, C_fg].  Slots past n_kept are zero.  Components are ordered by voxel
 * count descending, ties by label descending.  No host synchronisation; deterministic.  The workspace covers the worst case (every voxel its own
 * component); 0 = unsupported arguments. */
size_t mdt_seg_components_workspace_bytes(int n, int y, int x, int z, int n_seg_classes, int n_fg_classes, int k, int dim);
int mdt_seg_components(const float *logits, const long long *strides3, int n, int y, int x, int z, int n_seg_classes, int n_fg_classes, int k, int dim,
                       int median, unsigned char *seg_pred, int *comp_label, int *boxes, float *scores, int *n_kept, void *ws, size_t ws_bytes,
                       void *stream);
/* Class loss with stochastic hard-example mining.  replaces: compute_class_loss (models/retina_unet.py:126-164) / compute_rpn_class_loss
 * (models/mrcnn.py:176-213) incl. mutils.shem (utils/model_utils.py:674-691): softmax over all anchors, sort of the negatives' max foreground
 * probability, randperm sample, two cross-entropies.  logits [n_anchors, n_classes] contiguous fp32, matches int32 (-1 negative, 0 neutral,
 * > 0 positive class); pos_ids = the first n_pos_list positive anchor ids (int64, ascending; at most k_pos are used); k_pool = size of the
 * candidate pool (<= 1024, = shem_poolsize * k_pos), k_neg <= k_pool sampled negatives at most; rand_keys [k_pool] uniform [0,1) floats from the
 * caller's generator (the negative_count = max(1, #positives) pool members with the smallest keys are the sample).
 * Outputs (device): loss[1] = (CE_pos + CE_neg) / 2; neg_ix [k_neg] int64 = rank of each sampled negative inside the negative subset (-1 pad);
 * sel_rows / sel_labels / sel_w [k_pos + k_neg] = the rows entering the loss, their labels and weights (for the backward).
 * backward: grad_logits [n_anchors, n_classes] is zero-filled, then rows += grad_loss * w * (softmax - onehot). */
size_t mdt_shem_workspace_bytes(int n_anchors, int k_pool);
int mdt_shem_class_loss_forward(const float *logits, const int *matches, int n_anchors, int n_classes, const long long *pos_ids, int n_pos_list, int k_pos,
                                int k_pool, int k_neg, int shem_poolsize, const float *rand_keys, float *loss, long long *neg_ix, int *sel_rows,
                                int *sel_labels, float *sel_w, void *ws, size_t ws_bytes, void *stream);
int mdt_shem_class_loss_backward(const float *logits, int n_anchors, int n_classes, const int *sel_rows, const int *sel_labels, const float *sel_w,
                                 int n_sel, const float *grad_loss, float *grad_logits, void *stream);

/* ------------------------------------------------------------- inference-side consolidation (csrc/consolidate.cu) ----------------------------
 * replaces: weighted_box_clustering(dets, box_patch_id, thresh, n_ens) of predictor.py:597-706 (numpy loop per patient and class).
 * dets [n, 2*dim + 3] fp64 rows = (y1, x1, y2, x2, (z1, z2), score, patch-centre factor, number of overlapping patches); patch_id [n] int32 in
 * [0, n_patches) (the caller maps the reference's patch-id strings to dense ints); order [n] int32 = box indices by descending score.
 * Outputs (device): keep_scores [<= n], keep_coords [<= n, 2*dim] in cluster order, n_keep[1].  One resident CTA runs the whole greedy loop. */
size_t mdt_wbc_workspace_bytes(int n, int n_patches);
int mdt_wbc(const double *dets, const int *patch_id, const int *order, int n, int dim, int n_patches, double thresh, double n_ens, double *keep_scores,
            double *keep_coords, int *n_keep, void *ws, size_t ws_bytes, void *stream);
/* replaces: nms_2to3D(dets, thresh) of predictor.py:710-773.  dets [n, 6] fp64 rows = (y1, x1, y2, x2, score, slice id), slice ids in
 * [0, n_slices); order as above.  Outputs: keep [<= n] int64 indices of the cluster cores, keep_z [<= n, 2] = (z1, z2), n_keep[1]. */
size_t mdt_nms_2to3d_workspace_bytes(int n, int n_slices);
int mdt_nms_2to3d(const double *dets, const int *order, int n, double thresh, int n_slices, long long *keep, double *keep_z, int *n_keep, void *ws,
                  size_t ws_bytes, void *stream);

/* ------------------------------------------------------------- normalisation and activation (csrc/norm_act.cu) ------------------------------
 * replaces: nn.InstanceNorm{2,3}d, nn.BatchNorm{2,3}d and nn.LeakyReLU built by NDConvGenerator (utils/model_utils.py:739-781) for cf.norm /
 * cf.relu, and the add + activation after a normalised ResBlock conv3 (models/backbone.py:195-206).
 * x [n, s, c] fp32 channels-last (s voxels, any c >= 1).  per_sample = 1: groups (n, c) over s (instance norm; mean / rstd hold n*c values);
 * per_sample = 0: groups c over n*s (batch norm; c values).  mean / rstd = per-group mean and 1 / sqrt(biased variance + eps).
 * Reductions are fixed-order fp64 sums (no atomics): bit-identical from run to run.  Pointers need 4-byte alignment only (views may start
 * anywhere); the workspace 16 bytes.  act: 0 none, 1 ReLU, 2 leaky ReLU with negative slope `slope`.
 * mdt_norm_stats: batch statistics; with running_mean / running_var (per_sample = 0 and n*s >= 2 only) also running = (1 - momentum) * running
 * + momentum * stat, the variance unbiased (M / (M - 1)); num_batches_tracked (optional, int64) += 1.
 * mdt_norm_eval_stats: mean / rstd from the running statistics (batch norm in eval mode).
 * mdt_norm_apply: y = act((x - mean) * rstd * gamma + beta (+ residual)); gamma, beta, residual optional (NULL).
 * mdt_norm_backward: g = dy * act'(y) from the saved output (y > 0 -> 1, else 0 / slope); xhat = (x - mean) * rstd;
 * batch_stats = 1: dx = gamma * rstd * (g - sum g / M - xhat * sum(g xhat) / M) per group; batch_stats = 0 (running statistics): dx = g * gamma * rstd.
 * dgamma = sum g xhat, dbeta = sum g over each channel (optional); dresidual = g (optional).  The workspace is needed only when batch_stats or
 * dgamma / dbeta are set.  mdt_norm_workspace_bytes covers both passes; 0 = unsupported arguments.
 * mdt_act_forward / mdt_act_backward: y = act(x), dx = dy * act'(y) over `count` contiguous elements. */
size_t mdt_norm_workspace_bytes(int n, long long s, int c, int per_sample);
int mdt_norm_stats(const float *x, int n, long long s, int c, int per_sample, float eps, float momentum, float *mean, float *rstd,
                   float *running_mean, float *running_var, long long *num_batches_tracked, void *ws, size_t ws_bytes, void *stream);
int mdt_norm_eval_stats(const float *running_mean, const float *running_var, int c, float eps, float *mean, float *rstd, void *stream);
int mdt_norm_apply(const float *x, const float *mean, const float *rstd, const float *gamma, const float *beta, const float *residual, int n,
                   long long s, int c, int per_sample, int act, float slope, float *y, void *stream);
int mdt_norm_backward(const float *dy, const float *y, const float *x, const float *mean, const float *rstd, const float *gamma, int n, long long s,
                      int c, int per_sample, int act, float slope, int batch_stats, float *dx, float *dgamma, float *dbeta, float *dresidual, void *ws,
                      size_t ws_bytes, void *stream);
/* Batch norm over a batch split across ranks (per_sample = 0 semantics, x [n, s, c] as above).  mdt_norm_sample_sums: sums (device, [n][c]
 * double pairs (sum x, sum x^2), 16-byte aligned) of each sample; a sample's row split depends on (s, c) only, so its sums are bit-identical in a
 * batch of any size.  mdt_norm_stats_from_sums: rows [n_total][c] (all ranks' rows, rank-major) added in row order -> mean / rstd over
 * M = n_total * s, and the running statistics (unbiased with that M; n_total * s >= 2) and num_batches_tracked as mdt_norm_stats.
 * mdt_norm_backward_sample_sums: per-sample (sum g, sum g xhat) with g = dy * act'(y), as mdt_norm_backward.  mdt_norm_backward_from_sums: dx
 * with the totals of global_sums [n_total][c] and M = n_total * s; dgamma / dbeta = the sums of this rank's rows [local_first_row,
 * local_first_row + n) in order; dresidual = g.  Workspace (every sample-sum entry point and the from-sums backward):
 * mdt_norm_sample_workspace_bytes, 0 = unsupported arguments. */
size_t mdt_norm_sample_workspace_bytes(int n, long long s, int c);
int mdt_norm_sample_sums(const float *x, int n, long long s, int c, double *sums, void *ws, size_t ws_bytes, void *stream);
int mdt_norm_stats_from_sums(const double *sums, int n_total, long long s, int c, float eps, float momentum, float *mean, float *rstd,
                             float *running_mean, float *running_var, long long *num_batches_tracked, void *stream);
int mdt_norm_backward_sample_sums(const float *dy, const float *y, const float *x, const float *mean, const float *rstd, int n, long long s, int c,
                                  int act, float slope, double *sums, void *ws, size_t ws_bytes, void *stream);
int mdt_norm_backward_from_sums(const float *dy, const float *y, const float *x, const float *mean, const float *rstd, const float *gamma,
                                const double *global_sums, int n_total, int local_first_row, int n, long long s, int c, int act, float slope, float *dx,
                                float *dgamma, float *dbeta, float *dresidual, void *ws, size_t ws_bytes, void *stream);
int mdt_act_forward(const float *x, long long count, int act, float slope, float *y, void *stream);
int mdt_act_backward(const float *dy, const float *y, long long count, int act, float slope, float *dx, void *stream);

/* ------------------------------------------------------------- training-batch augmentation (csrc/augment.cu) -------------------------------
 * replaces: the MirrorTransform -> SpatialTransform -> ConvertSegToBoundingBoxCoordinates chain of batchgenerators 0.19.3 that
 * experiments/{lidc_exp,toy_exp}/data_loader.py run in CPU worker processes.  Spatial axes are (y, x, z); 2D: z absent (shape arrays hold dim
 * entries).  All three ops are deterministic (integer atomics only).
 *
 * Elastic field.  replaces: scipy.ndimage.gaussian_filter(noise, sigma, mode='constant', cval=0) * alpha of batchgenerators'
 * elastic_deform_coordinates (augmentations/utils.py).  noise / out [n, *shape] fp64, n fields; field f is filtered with sigma_host[f] (radius
 * int(4 sigma + 0.5) <= 200, else MDT_EUNSUPPORTED; weights normalised in fp64 as scipy does) and multiplied by scale_host[f].  n <= 1024. */
size_t mdt_augment_gaussian_workspace_bytes(int dim, int n, const int *shape_host);
int mdt_augment_gaussian(int dim, const double *noise, int n, const int *shape_host, const double *sigma_host, const double *scale_host, double *out,
                         void *ws, size_t ws_bytes, void *stream);
/* Spatial transform.  replaces: MirrorTransform + SpatialTransform (augmentations/spatial_transformations.py augment_spatial) with
 * order_data = 3, border_mode_data = 'nearest', order_seg = 0, border_mode_seg = 'constant', cval 0.
 * Output voxel i of element b samples the source at q = (i - (P - 1) / 2 + elastic[b, :, i]) . m + centre (fp64, row vector times m), in the
 * frame of the source mirrored on every axis with flip[d] != 0.  data [n, c, *src] fp32 -> data_out [n, c, *patch]: scipy's
 * map_coordinates(order=3, mode='nearest', prefilter=True), from cubic B-spline coefficients the call writes into the workspace.
 * seg [n, 1, *src] uint8 -> seg_out [n, 1, *patch]: map_coordinates(order=0, mode='constant', cval=0), i.e. 0 where q_d < 0 or q_d > S_d - 1 on
 * any axis, else the id at floor(q + 0.5).  seg and seg_out are both NULL or both set.  params: device array of n blocks; elastic: device
 * [n, dim, *patch] fp64 displacement (alpha already applied), NULL = none.  The source size is the batch array's. */
typedef struct mdt_augment_params {
    double m[9];       /* row-major 3x3 (2D: the upper-left 2x2) rotation with the scale folded in */
    double centre[3];  /* crop centre in source voxels */
    int flip[3];       /* mirror the source along this axis */
    int pad_;
} mdt_augment_params;
size_t mdt_augment_spatial_workspace_bytes(int dim, int n, int c, const int *src_host);
int mdt_augment_spatial(int dim, const float *data, const unsigned char *seg, int n, int c, const int *src_host, const int *patch_host,
                        const mdt_augment_params *params, const double *elastic, float *data_out, unsigned char *seg_out, void *ws, size_t ws_bytes,
                        void *stream);
/* Seg to boxes.  replaces: ConvertSegToBoundingBoxCoordinates (get_rois_from_seg_flag=False) of augmentations/utils.py
 * convert_seg_to_bounding_box_coordinates.  seg [n, 1, *patch] uint8 instance ids; lut [n, 256] uint8 maps each id to its output label
 * (lut[b][0] = 0).  Outputs: stats [n, 255, 7] int32 per (element, id 1..255) = voxel count, min y/x/z, max y/x/z (count 0: min INT_MAX, max
 * -1; 2D: z entries 0); seg_out [n, 1, *patch] = lut applied; masks (optional, NULL to skip) [n, n_mask_ids, *patch] uint8 = (seg == k) for
 * k = 1..n_mask_ids.  No workspace. */
int mdt_augment_seg_to_boxes(int dim, const unsigned char *seg, int n, const int *patch_host, const unsigned char *lut, int n_mask_ids, int *stats,
                             unsigned char *seg_out, unsigned char *masks, void *stream);
/* ROIs from connected components (csrc/seg_rois.cu).  replaces: ConvertSegToBoundingBoxCoordinates(get_rois_from_seg_flag=True) of
 * convert_seg_to_bounding_box_coordinates, as experiments/pet_ct_tnm_classification/data_loader.py calls it (scipy.ndimage.label per element).
 * seg [n, 1, *shape] uint8; foreground = seg != 0 whatever the value.  Components: face-connected (6 neighbours in 3D, 4 in 2D) within one
 * element, numbered in scipy.ndimage.label's order (first voxel in C order), consecutively over the batch: element b owns ids
 * elem_first[b] .. elem_first[b + 1] - 1, elem_first[n] = total.  No cap on the number of components.  Outputs (device):
 * comp_label int32 [n, *shape] = component id or -1; elem_first int32 [n + 1]; stats int32 [n * ceil(V / 2), 7] (V = voxels per element, the
 * most components an element can have; entries past elem_first[n] untouched) = per component voxel count, min y/x/z, max y/x/z (2D: z 0);
 * seg_out [n, 1, *shape] uint8 = (seg != 0) without class_specific, else class_target[b] + 1 where 1 <= seg <= n_b (the element's
 * component count) and seg elsewhere.  class_target: device int32 [n], read only with class_specific.  n * V < 2^31, else MDT_EUNSUPPORTED.
 * Deterministic (integer atomics only), no host synchronisation.  Workspace: 8 bytes per voxel plus the scan's temporary storage. */
size_t mdt_seg_rois_workspace_bytes(int dim, int n, const int *shape_host);
int mdt_seg_rois(int dim, const unsigned char *seg, int n, const int *shape_host, const int *class_target, int class_specific, int *comp_label,
                 int *elem_first, int *stats, unsigned char *seg_out, void *ws, size_t ws_bytes, void *stream);
/* masks [n_comp, *shape] uint8 = (comp_label == k) within component k's element, for the first n_comp component ids of an mdt_seg_rois call's
 * comp_label / elem_first (device).  n_comp is elem_first[n] read back by the caller; 0 writes nothing. */
int mdt_seg_rois_masks(int dim, const int *comp_label, int n, const int *shape_host, const int *elem_first, int n_comp, unsigned char *masks,
                       void *stream);

/* ------------------------------------------------------------- Mask R-CNN mask pasting (csrc/unmold.cu) -----------------------------------
 * replaces: the seg_preds loop of get_results (models/mrcnn.py:717-799) with unmold_mask_2D / unmold_mask_3D (utils/model_utils.py:147-183):
 * one scipy.ndimage.zoom(order=1) per detection on the host, pasted into a full-size volume, max over the element's volumes, np.round.
 * detections [n, 2*dim + 3] fp32 contiguous rows (y1, x1, y2, x2, (z1, z2), batch_ix, class_id, score); masks logical [n, n_classes,
 * *mask_shape] fp32 with element strides mask_strides_host[dim + 2] (NCDHW or channels-last).  A row belongs to element b iff batch_ix == b;
 * its box and class are truncated to int32 and it contributes iff every extent hi - lo > 0 and 0 <= class < n_classes.  The mask of its class
 * is resized as zoom(order=1, mode='constant') does (fp64, bit-identical to scipy) and pasted at [lo, lo + extent), intersected with the image:
 * a box with lo < 0 (refine_detections never makes one) is an interval, not numpy's negative slice.
 * Outputs: seg uint8 [batch, *img_shape] = round half to even of max(0, max over the rows covering the voxel), 0 where none does;
 * seg_float (optional, NULL to skip) fp32 [batch, *img_shape] = that maximum before rounding.  Every byte is written once; no workspace,
 * no atomics, deterministic. */
int mdt_unmold_masks(int dim, const float *detections, int n, const float *masks, const int64_t *mask_strides_host, int n_classes,
                     const int *mask_shape_host, int batch, const int *img_shape_host, unsigned char *seg, float *seg_float, void *stream);

/* ------------------------------------------------------------- evaluation (csrc/evaluate.cu) ----------------------------------------------
 * replaces: Evaluator.evaluate_predictions / return_metrics of evaluator.py:39-313 and get_roi_ap_from_df / compute_roi_ap :361-437
 * (numpy loops per IoU, class, patient and element; pandas filters; scikit-learn curves).  All fp64; results are bit-identical to numpy's.
 *
 * mdt_eval_match: boxes grouped by (element e, class index c), group g = e * n_classes + c.  cand_boxes [n_cand, 2*dim] / cand_scores
 * [n_cand] and gt_boxes [n_gt, 2*dim] in group order, with CSR offsets cand_offsets / gt_offsets [n_elem * n_classes + 1]; the elements
 * of patient p are [elem_offsets[p], elem_offsets[p + 1]).  match_ious [n_iou].  Rows are written in the reference's order (IoU, class,
 * patient, element; per element double-match FPs, TPs, unmatched FPs, FNs; one patient_tn row for a (IoU, class, patient) without rows):
 * row_score [max_rows] and row_meta [max_rows, 4] int32 (16-byte aligned) = (type 0 det_tp / 1 det_fp / 2 det_fn / 3 patient_tn, class
 * index, patient index, IoU index), n_rows [1].  max_rows = n_iou * (n_cand + n_gt + n_classes * n_patients) bounds n_rows.  A candidate
 * whose IoU row holds a NaN emits no row.  Workspace queries return 0 when the scan library cannot size its scratch (no device). */
size_t mdt_eval_match_workspace_bytes(int n_slots, int n_cand, int n_gt, int n_iou);
int mdt_eval_match(const double *cand_boxes, const double *cand_scores, const int *cand_offsets, int n_cand, const double *gt_boxes,
                   const int *gt_offsets, int n_gt, const int *elem_offsets, int n_patients, int n_classes, int dim, const double *match_ious,
                   int n_iou, double *row_score, int *row_meta, int *n_rows, void *ws, size_t ws_bytes, void *stream);
/* mdt_eval_roi_ap: rows (score, segment id in [0, n_seg) or -1, type code as above).  Per segment: all_p = rows of type 0 or 2; the
 * type-0/1 rows sorted by descending score (stable: ties keep row order; NaN scores are left out); for every threshold t the nd rows with
 * score > t give rc = tp / all_p and the reverse-max precision envelope, read at np.searchsorted(rc, recall_points, 'left').
 * Outputs: q [n_seg, n_thresh, n_recall] (0 past the last detection, and everywhere when all_p = 0), counts [n_seg, 1 + n_thresh] =
 * (all_p, nd per threshold).  n_recall <= 128. */
size_t mdt_eval_roi_ap_workspace_bytes(int n_rows, int n_seg);
int mdt_eval_roi_ap(const double *row_score, const int *row_seg, const int *row_kind, int n_rows, int n_seg, const double *thresholds,
                    int n_thresh, const double *recall_points, int n_recall, double *q, int *counts, void *ws, size_t ws_bytes, void *stream);
/* mdt_eval_patient: per slot (class, pid) the max label (0/1) and max score over the rows with row_slot = that slot (-1: no slot); a slot
 * without rows is not a patient.  Segment k holds the slots seg_slots[seg_offsets[k] .. seg_offsets[k + 1]) (n_members in all).  For
 * each segment, in descending order of its n_thr[k] distinct patient scores: thr, tps = positives with score >= thr, fps = negatives
 * with score >= thr (scikit-learn's binary_clf_curve counts), written from seg_offsets[k] on. */
size_t mdt_eval_patient_workspace_bytes(int n_slots, int n_members);
int mdt_eval_patient(const double *row_score, const int *row_label, const int *row_slot, int n_rows, int n_slots, const int *seg_offsets,
                     const int *seg_slots, int n_members, int n_seg, double *thr, int *tps, int *fps, int *n_thr, void *ws, size_t ws_bytes,
                     void *stream);
/* Patient bootstrap.  The units are P = n_patients patients; a row's patient index is in [0, P).  mult [n_boot, P] int32 holds one
 * resample per row, m[p] in [0, P] (the host draws it: numpy's RandomState([seed, b]).randint(0, P, P), bincount).  A resample's metrics
 * are by definition those of the materialised resample: every row of patient p repeated m[p] times in place (copies next to each other),
 * copy j of p a patient of its own, matching not redone.  The kernels never materialise it; every count is an integer sum of weights and
 * the outputs equal the evaluation of the materialised rows bit for bit (the argument is in csrc/evaluate.cu).  Both entries check the
 * patient indices and multiplicities on the device and wait for that check (one synchronisation of `stream`): MDT_EINVAL when one is out
 * of range, and also when n_patients * n_rows >= 2^31 (the bound on every weighted count), on negative sizes or n_recall / n_rates > 128.
 * n_boot = 0 does nothing.
 *
 * mdt_eval_bootstrap_roi: rows as mdt_eval_roi_ap's plus row_patient; one threshold (detections with score > threshold; NaN scores left
 * out); recall_points ascending.  Per (resample b, segment s), o = b * n_seg + s: q [o, n_recall] as mdt_eval_roi_ap's, counts [o, 2] =
 * (weighted all_p, weighted nd), froc_tp [o, n_rates] = max{TP(v) : FP(v) <= fp_limits[f]} over the operating points (origin and, per
 * distinct score v above the threshold, the weighted TP / FP detections with score >= v): the step FROC, no interpolation between points.
 * The sensitivity is froc_tp / all_p (all_p = det_tp + det_fn rows, the GT lesions); fp_limits [n_rates] = rate * P, fp64. */
size_t mdt_eval_bootstrap_roi_workspace_bytes(int n_rows, int n_seg, int n_patients);
int mdt_eval_bootstrap_roi(const double *row_score, const int *row_seg, const int *row_kind, const int *row_patient, int n_rows, int n_seg,
                           int n_patients, const int *mult, int n_boot, double threshold, const double *recall_points, int n_recall,
                           const double *fp_limits, int n_rates, double *q, int *counts, int *froc_tp, void *ws, size_t ws_bytes, void *stream);
/* mdt_eval_bootstrap_patient: rows, slots and segments as mdt_eval_patient's plus row_patient (the rows of one slot share a patient);
 * n_patients * n_members < 2^31.  Per resample b and segment k, the distinct thresholds with nonzero weight in descending order with the
 * weighted tps / fps at each, written from b * n_members + seg_offsets[k] on; n_thr [n_boot, n_seg]. */
size_t mdt_eval_bootstrap_patient_workspace_bytes(int n_slots, int n_members, int n_seg);
int mdt_eval_bootstrap_patient(const double *row_score, const int *row_label, const int *row_slot, const int *row_patient, int n_rows,
                               int n_slots, const int *seg_offsets, const int *seg_slots, int n_members, int n_seg, int n_patients,
                               const int *mult, int n_boot, double *thr, int *tps, int *fps, int *n_thr, void *ws, size_t ws_bytes,
                               void *stream);

/* ------------------------------------------------------------- data loader (csrc/loader.cu) -----------------------------------------------
 * replaces: the volume scans of BatchGenerator.generate_train_batch and the tiling of PatientBatchIterator.generate_train_batch in
 * experiments/{lidc_exp,toy_exp,pet_ct_tnm_classification}/data_loader.py (np.sum / np.unique / np.argwhere over the whole patient, np.pad,
 * np.take, the slice and patch crops).
 *
 * mdt_loader_fg_index: seg [z, y, x] uint8, one patient in the memory order of its .npy file, read as the transposed (y, x, z) view the
 * loaders work on.  counts [256] int32 = voxels per label (counts[0]: background).  order [cap] int32 = the (y, x, z) linear index
 * (y * x_ext + x) * z_ext + z of every foreground voxel, grouped by label (1 .. 255 ascending), each group in ascending index order (np.argwhere
 * of seg == label on the transposed view); entries at or past min(cap, number of foreground voxels) are not written.  cap = 0 (order may be
 * NULL) writes counts only.  z <= 6000 and z * y * x < 2^31, else MDT_EUNSUPPORTED.  Deterministic.  Workspace: 1 KiB per 32-column tile of
 * a y row. */
size_t mdt_loader_fg_index_workspace_bytes(int z, int y, int x);
int mdt_loader_fg_index(const unsigned char *seg, int z, int y, int x, int *counts, int *order, int cap, void *ws, size_t ws_bytes, void *stream);
/* mdt_loader_gather: out [n, c, i, j, k] (out_dtype) = src_b[tab_c[b, c], tab_z[b, c, k], tab_y[b, i], tab_x[b, j]] where src_b is element
 * b's [c, z, y, x] volume (src_dtype) at element offset elems[b].offset of src; a table entry outside [0, extent) of its axis (-1 by
 * convention) gives 0.  Converts as numpy's astype does (float -> uint8 truncates; fp64 -> fp16 rounds once).  k > 1: i <= 65535 and n * c <=
 * 65535, else MDT_EUNSUPPORTED.  Tables are device int32 arrays.  No workspace. */
#define MDT_DTYPE_U8 0
#define MDT_DTYPE_F16 1
#define MDT_DTYPE_F32 2
#define MDT_DTYPE_F64 3
#define MDT_DTYPE_I16 4
typedef struct mdt_loader_src {
    long long offset;  /* in elements of src_dtype */
    int c, z, y, x;    /* the element's source extents */
} mdt_loader_src;
int mdt_loader_gather(int src_dtype, const void *src, const mdt_loader_src *elems, int n, int c, int i, int j, int k, const int *tab_c, const int *tab_z,
                      const int *tab_y, const int *tab_x, int out_dtype, void *out, void *stream);

/* ------------------------------------------------------------- LIDC preprocessing (csrc/preprocess.cu) ------------------------------------
 * replaces: the skimage.transform.resize calls (scikit-image 0.16.2: order 1, mode 'edge', anti_aliasing on, clip) and the numpy CT
 * normalisation and rater vote of experiments/lidc_exp/preprocessing.py (resample_array, pp_patient).  Volumes are (z, y, x), C order.
 * Every call is asynchronous on `stream` and deterministic (no atomics).
 *
 * mdt_pp_resample: out [out_shape] fp32 = resize(src [in_shape] as fp64): with factors f = in / out per axis, scipy's gaussian_filter at
 * sigma = max(0, (f - 1) / 2) with mode 'nearest' on the axes with sigma > 1e-15 (fp64 weights, radius int(4 sigma + 0.5) <= 64, else
 * MDT_EUNSUPPORTED), then map_coordinates(order=1, mode='nearest') at f (j + 0.5) - 0.5 in fp64, rounded once to fp32.  src_dtype:
 * MDT_DTYPE_U8, MDT_DTYPE_I16 or MDT_DTYPE_F32.  Workspace: one fp64 volume of in_shape per blurred axis, at most two (0 bytes when no
 * axis is blurred, ws may then be NULL). */
size_t mdt_pp_resample_workspace_bytes(const int *in_shape, const int *out_shape);
int mdt_pp_resample(int src_dtype, const void *src, const int *in_shape, const int *out_shape, float *out, void *ws, size_t ws_bytes, void *stream);
/* mdt_pp_normalize: x [n] fp32 in place: clip to [-1200, 600], mean and population std of the clipped values in fp64 (fixed 1024-way
 * partial sums and fixed trees), then x = fl32(fl32(x - fl32(mean)) / fp16(fl32(std))).  stats [2] fp64 (device) = {mean, std} before
 * rounding.  Workspace: 8 KiB. */
size_t mdt_pp_normalize_workspace_bytes(long long n);
int mdt_pp_normalize(float *x, long long n, double *stats, void *ws, size_t ws_bytes, void *stream);
/* mdt_pp_vote_add: acc [n] fp32 = first ? rater : acc + rater (the raters of one ROI summed in fp32 in call order). */
int mdt_pp_vote_add(float *acc, const float *rater, long long n, int first, void *stream);
/* mdt_pp_vote_label: the vote of ROI `roi` (0-based, <= 254, else MDT_EUNSUPPORTED): where acc / max(4, n_raters) >= 0.5 (fp32 division),
 * labels [n] uint8 = 1 + the number of ROIs r < roi with kept[r] != 0; kept [>= roi + 1] int32: kept[roi] = 1 if any voxel was labelled, else
 * 0 (kept[0 .. roi) are read).  roi 0 writes every voxel of labels (0 where its vote is below 0.5); later ROIs overwrite. */
int mdt_pp_vote_label(const float *acc, long long n, int n_raters, int roi, unsigned char *labels, int *kept, void *stream);
/* mdt_pp_label_summary: labels [z, plane] uint8 -> slice_nz [z] uint8 = any voxel of the slice != 0, present [256] uint8 = label occurs. */
int mdt_pp_label_summary(const unsigned char *labels, int z, long long plane, unsigned char *slice_nz, unsigned char *present, void *stream);

/* ------------------------------------------------------------- PET-CT preprocessing (csrc/petct_preprocess.cu) -----------------------------
 * replaces: the SimpleITK resampling, the segment merge, get_z_crops' per-slice scan (clear_border, scipy.ndimage.label, center_of_mass) and
 * the two-channel normalisation of experiments/pet_ct_tnm_classification/preprocessing.py.  Volumes are (z, y, x), C order, unless strides
 * say otherwise.  Every call is asynchronous on `stream` and deterministic.
 *
 * mdt_petct_grid: an ITK image geometry in ITK's (x, y, z) axis order: size, origin, spacing (> 0) and the row-major 3x3 direction.
 * mdt_petct_resample: out (out_grid) = ResampleImageFilter of src (in_grid) with the identity transform and linear interpolation, per voxel in
 * fp64: p = origin_o + sum_c (direction_o[r][c] spacing_o[c]) i_c, then c_r = sum_k (direction_i[k][r] / spacing_i[r]) (p_k - origin_i[k]),
 * each sum taken in axis order without contraction.  A point with some c_r outside [-0.5, size_r - 0.5) gets 0; otherwise base = max(0,
 * floor(c)), and per axis (x, then y, then z) a + (b - a) d with d = c - base (the base sample alone where d <= 0 or base + 1 is past the
 * end).  The value is clamped to out_dtype's range and truncated (MDT_DTYPE_U8, MDT_DTYPE_I16) or rounded (MDT_DTYPE_F32).  src_dtype and
 * out_dtype: MDT_DTYPE_U8, MDT_DTYPE_I16 or MDT_DTYPE_F32, else MDT_EINVAL.  No workspace. */
typedef struct mdt_petct_grid {
    int size[3];
    double origin[3];
    double spacing[3];
    double direction[9];
} mdt_petct_grid;
int mdt_petct_resample(int src_dtype, const void *src, const mdt_petct_grid *in_grid, int out_dtype, void *out, const mdt_petct_grid *out_grid,
                       void *stream);
/* mdt_petct_seg_merge: out [z, y, x] uint8 = 1 where some segment k with selected[k] != 0 (host uint8 [n_seg]) has segs[k, x, y, z] == 1,
 * else 0.  segs: device, src_dtype as for mdt_petct_resample, element strides (host int64 [4], >= 0) of its axes (k, x, y, z).  n_seg <= 256,
 * else MDT_EUNSUPPORTED.  No workspace. */
int mdt_petct_seg_merge(int src_dtype, const void *segs, int n_seg, int x, int y, int z, const long long *strides, const unsigned char *selected,
                        unsigned char *out, void *stream);
/* mdt_petct_body_components: per z slice of ct [z, y, x] (src_dtype as above), the pixels with value < -600, without the 8-connected
 * components that own a pixel of the slice's one-pixel border (skimage's clear_border), labelled with 4-connectivity (scipy.ndimage.label)
 * and numbered over the volume in C order of their first pixel.  label [z, y, x] int32: the component id or -1; slice_first [z + 1] int32:
 * slice s owns ids slice_first[s] .. slice_first[s + 1] - 1; stats [stats_cap, 3] int64: (pixel count, sum of rows, sum of columns) per id,
 * rows past slice_first[z] unwritten.  stats_cap >= mdt_petct_body_components_capacity(z, y, x) = z * ceil(y x / 2), else MDT_EINVAL;
 * z y x < 2^31, else MDT_EUNSUPPORTED (both queries return 0 then).  Integer atomics only. */
long long mdt_petct_body_components_capacity(int z, int y, int x);
size_t mdt_petct_body_components_workspace_bytes(int z, int y, int x);
int mdt_petct_body_components(int src_dtype, const void *ct, int z, int y, int x, int *label, int *slice_first, long long *stats, long long stats_cap,
                              void *ws, size_t ws_bytes, void *stream);
/* mdt_petct_zcrop_criterion: flags [z] uint8 = 1 where the slice has at least n_comps components of mdt_petct_body_components with count >
 * min_pix and (rows / count - y / 2)^2 + (cols / count - x / 2)^2 < rad_crit, each operation rounded separately in fp64.  No workspace. */
int mdt_petct_zcrop_criterion(const int *slice_first, const long long *stats, int z, int y, int x, long long min_pix, int n_comps, double rad_crit,
                              unsigned char *flags, void *stream);
/* mdt_petct_normalize: out [2, n] fp32 from the cropped CT ct [n] int16 and PET pet [n] fp32.  CT: c = (1200 + clip(x, -1200, 600)) / 1800,
 * its mean and population std in fp64, out[0] = fl32((c - mean) / std) in fp64.  PET: mean and population std in fp64, each rounded to fp32,
 * out[1] = fl32(fl32(p - mean) / std).  stats [4] fp64 (device) = {CT mean, CT std, PET mean, PET std} before rounding.  The sums run over
 * fixed 1024-way partial sums and fixed trees.  Workspace: 16 KiB. */
size_t mdt_petct_normalize_workspace_bytes(long long n);
int mdt_petct_normalize(const short *ct, const float *pet, long long n, float *out, double *stats, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------- toy experiment images (csrc/toys.cu) ----------------------------------------
 * replaces: multi_processing_create_image of experiments/toy_exp/generate_toys.py, with a per-image seed in place of numpy's global state.
 *
 * mdt_toy_images: image b draws from numpy's legacy RandomState seeded by init_by_array on keys [b, 0 .. 2] (device uint32 [n, 3]), with
 * the reference's calls in its order: rand(320, 320), then cx = randint(margin, 320 - margin), cy = randint(margin, 320 - margin),
 * class_id = randint(0, 2).  Where (x - cx)^2 + (y - cy)^2 < r^2 (x the column, y the row, r = radius0 / radius1 by class_id) it adds 0.2
 * to the image and sets seg to 1; with MDT_TOY_HOLE and class_id 1 it then subtracts 0.2 where the distance is below 4, and with
 * MDT_TOY_HOLE_CLEARS_SEG also sets seg to 0 there.  img: device fp64 [n, 2, 320, 320] (image plane, then seg as 0.0 / 1.0), the array the
 * reference saves; params: device int32 [n, 3] = (cx, cy, class_id).  0 <= margin < 320 - margin, radii >= 0, else MDT_EINVAL.  One CTA per
 * image; the bound is the 1.64 MB written per image and the 329 dependent twists of its MT19937 state.  No workspace; deterministic. */
#define MDT_TOY_HOLE 1
#define MDT_TOY_HOLE_CLEARS_SEG 2
int mdt_toy_images(const uint32_t *keys, int n, int margin, int radius0, int radius1, int flags, double *img, int *params, void *stream);

/* ------------------------------------------------------------- plot rendering (csrc/render.cu) ---------------------------------------------
 * replaces: the matplotlib drawing behind plotting.py (imshow, plot, hist, text, savefig's rasteriser); the host (plotting.py) builds the
 * scene and maps data to integer pixels, these draw it into canvas, a device uint8 [height, width, 3] the caller fills (white) first.
 *
 * mdt_render_panel: one image source and where it goes.  src: device pointer to element (0, 0) of an [h, w] view with element strides
 * stride_y, stride_x; dtype MDT_DTYPE_U8, MDT_DTYPE_F16 or MDT_DTYPE_F32.  Source (r, c) fills [y0 + r s, y0 + (r + 1) s) x
 * [x0 + c s, x0 + (c + 1) s) of the canvas (s = scale >= 1), clipped to it; panels must not overlap.  A descriptor with another dtype or
 * mode, h, w or scale < 1 draws nothing.
 * mdt_render_panel_range: range [n, 2] fp32 (device) = (lo, hi) over the finite values of each panel's source, lo = hi = 0 when it has none.
 * mdt_render_panels: MDT_RENDER_GREY writes g = min(255, (int)fl(fl(x - lo) / fl(hi - lo)) * 256) (each operation rounded to fp32) as
 * (g, g, g), or 0 when hi <= lo, from range [n, 2]; MDT_RENDER_CLASS writes palette[clamp((int)x, 0, n_palette - 1)] (device uint8
 * [n_palette, 3], n_palette >= 1).  Non-finite values keep the canvas.  n <= 65535, else MDT_EUNSUPPORTED.  panels: device array.
 * mdt_render_prim: kind MDT_PRIM_SEGMENT: (x0, y0) -> (x1, y1), both ends drawn; x-major (|dx| >= |dy|) pixels are
 * (x, y0 + sgn(dy) floor((2 |dy| t + |dx|) / (2 |dx|))) at step t = |x - x0| (y-major symmetric); with dash_period > 0 only the steps with
 * (dash_offset + t) mod dash_period < dash_on (dash_on >= 1, dash_offset >= 0).  MDT_PRIM_RECT: [x0, x1) x [y0, y1) blended as
 * (alpha c + (256 - alpha) dst + 128) >> 8 per channel, 0 <= alpha <= 256.  MDT_PRIM_GLYPH: character code (33 .. 126) of the library's
 * 6 x 8 bitmap font with its top-left at (x0, y0), each font pixel a scale x scale block.  rgb = 0xRRGGBB.  A primitive with a coordinate
 * beyond +-2^24 or an argument outside these ranges draws nothing.
 * mdt_render_prims: draws prims [n_prims] (device) strictly in list order, the last to cover a pixel wins (alpha rectangles blend over
 * what is there), clipped to the canvas.  ceil(height / 16) <= 65535, else MDT_EUNSUPPORTED.  No atomics: deterministic.  No workspace. */
#define MDT_RENDER_GREY 0
#define MDT_RENDER_CLASS 1
#define MDT_PRIM_SEGMENT 0
#define MDT_PRIM_RECT 1
#define MDT_PRIM_GLYPH 2
typedef struct mdt_render_panel {
    const void *src;
    long long stride_y, stride_x;
    int dtype, h, w, y0, x0, scale, mode, pad;
} mdt_render_panel;
typedef struct mdt_render_prim {
    int kind, x0, y0, x1, y1, rgb, alpha, code, scale, dash_on, dash_period, dash_offset;
} mdt_render_prim;
int mdt_render_panel_range(const mdt_render_panel *panels, int n_panels, float *range, void *stream);
int mdt_render_panels(const mdt_render_panel *panels, int n_panels, const float *range, const unsigned char *palette, int n_palette,
                      unsigned char *canvas, int height, int width, void *stream);
int mdt_render_prims(const mdt_render_prim *prims, int n_prims, unsigned char *canvas, int height, int width, void *stream);

/* number of kernel launches issued by this library since load (all entry points) — feeds bench.py's gpu_launches */
unsigned long long mdt_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* MDT_B200_H */
