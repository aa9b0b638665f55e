"""Inference-side box consolidation on libmdt_b200 (csrc/consolidate.cu) behind the call surface of the reference's predictor.py:

  weighted_box_clustering(dets, box_patch_id, thresh, n_ens)   predictor.py:597-706
  nms_2to3D(dets, thresh)                                      predictor.py:710-773
  apply_wbc_to_patient(inputs)                                 predictor.py:513-549
  merge_2D_to_3D_preds_per_patient(inputs)                     predictor.py:553-593

Same arguments (numpy arrays / lists of box dicts) and return values as the reference, so `Predictor` can call them unchanged; the greedy cluster
loops run in one kernel each on the current CUDA device (fp64, the reference's expression order).  No CPU fallback.
"""
import io
import pickle
import sys

import numpy as np
import torch

from . import _lib as L


def _device():
    if not torch.cuda.is_available():
        raise L.MdtError("libmdt_b200 consolidation ops need a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def weighted_box_clustering(dets, box_patch_id, thresh, n_ens):
    """dets (n, (y1, x1, y2, x2, (z1), (z2), score, box_pc_fact, box_n_ov)), box_patch_id (n,) any hashable dtype
    -> (keep_scores: list of float, keep_coords: list of [y1, x1, y2, x2, (z1, z2)])"""
    dets = np.ascontiguousarray(dets, dtype=np.float64)
    n = dets.shape[0]
    if n == 0:
        return [], []
    dim = 2 if dets.shape[1] == 7 else 3
    lib = L.load()
    dev = _device()
    _, dense = np.unique(np.asarray(box_patch_id), return_inverse=True)
    n_patches = int(dense.max()) + 1
    d = torch.from_numpy(dets).to(dev)
    pid = torch.from_numpy(dense.astype(np.int32)).to(dev)
    order = torch.sort(d[:, -3], descending=True, stable=True)[1].to(torch.int32)
    scores = torch.empty(n, dtype=torch.float64, device=dev)
    coords = torch.empty((n, 2 * dim), dtype=torch.float64, device=dev)
    n_keep = torch.zeros(1, dtype=torch.int32, device=dev)
    ws_bytes = lib.mdt_wbc_workspace_bytes(n, n_patches)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.mdt_wbc(L.ptr(d), L.ptr(pid), L.ptr(order), n, dim, n_patches, float(thresh), float(n_ens), L.ptr(scores), L.ptr(coords), L.ptr(n_keep),
                            L.ptr(ws), ws_bytes, L.stream_ptr()))
    k = int(n_keep.item())
    return scores[:k].cpu().tolist(), coords[:k].cpu().tolist()


def nms_2to3D(dets, thresh):
    """dets (n, (y1, x1, y2, x2, score, slice_id)) -> (keep: list of indices, keep_z: list of [z1, z2])"""
    dets = np.ascontiguousarray(dets, dtype=np.float64)
    n = dets.shape[0]
    if n == 0:
        return [], []
    lib = L.load()
    dev = _device()
    if dets[:, -1].min() < 0:
        raise L.MdtError("nms_2to3D: slice ids must be non-negative")
    n_slices = int(dets[:, -1].max()) + 1
    d = torch.from_numpy(dets).to(dev)
    order = torch.sort(d[:, -2], descending=True, stable=True)[1].to(torch.int32)
    keep = torch.empty(n, dtype=torch.int64, device=dev)
    keep_z = torch.empty((n, 2), dtype=torch.float64, device=dev)
    n_keep = torch.zeros(1, dtype=torch.int32, device=dev)
    ws_bytes = lib.mdt_nms_2to3d_workspace_bytes(n, n_slices)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.mdt_nms_2to3d(L.ptr(d), L.ptr(order), n, float(thresh), n_slices, L.ptr(keep), L.ptr(keep_z), L.ptr(n_keep), L.ptr(ws), ws_bytes,
                                  L.stream_ptr()))
    k = int(n_keep.item())
    return keep[:k].cpu().tolist(), keep_z[:k].cpu().tolist()


def apply_wbc_to_patient(inputs):
    """(in_patient_results_list, pid, class_dict, wcs_iou, n_ens) -> [out_patient_results_list, pid]   (predictor.py:513-549)"""
    in_patient_results_list, pid, class_dict, wcs_iou, n_ens = inputs
    out_patient_results_list = [[] for _ in range(len(in_patient_results_list))]
    for bix, b in enumerate(in_patient_results_list):
        for cl in list(class_dict.keys()):
            boxes = [box for box in b if (box['box_type'] == 'det' and box['box_pred_class_id'] == cl)]
            if len(boxes) == 0:
                continue
            dets = np.concatenate((np.array([bx['box_coords'] for bx in boxes]),
                                   np.array([bx['box_score'] for bx in boxes])[:, None],
                                   np.array([bx['box_patch_center_factor'] for bx in boxes])[:, None],
                                   np.array([bx['box_n_overlaps'] for bx in boxes])[:, None]), axis=1)
            keep_scores, keep_coords = weighted_box_clustering(dets, np.array([bx['patch_id'] for bx in boxes]), wcs_iou, n_ens)
            for sc, co in zip(keep_scores, keep_coords):
                out_patient_results_list[bix].append({'box_type': 'det', 'box_coords': co, 'box_score': sc, 'box_pred_class_id': cl})
        out_patient_results_list[bix].extend([box for box in b if box['box_type'] == 'gt'])
    return [out_patient_results_list, pid]


def merge_2D_to_3D_preds_per_patient(inputs):
    """(in_patient_results_list, pid, class_dict, merge_3D_iou) -> [[boxes], pid]: slices in the batch dimension -> cubes (predictor.py:553-593)"""
    in_patient_results_list, pid, class_dict, merge_3D_iou = inputs
    out_patient_results_list = []
    for cl in list(class_dict.keys()):
        boxes, slice_ids = [], []
        for bix, b in enumerate(in_patient_results_list):
            det_boxes = [box for box in b if (box['box_type'] == 'det' and box['box_pred_class_id'] == cl)]
            boxes += det_boxes
            slice_ids += [bix] * len(det_boxes)
        if len(boxes) == 0:
            continue
        box_coords = np.array([bx['box_coords'] for bx in boxes])
        box_scores = np.array([bx['box_score'] for bx in boxes])
        keep_ix, keep_z = nms_2to3D(np.concatenate((box_coords, box_scores[:, None], np.array(slice_ids)[:, None]), axis=1), merge_3D_iou)
        for kix, kz in zip(keep_ix, keep_z):
            out_patient_results_list.append({'box_type': 'det', 'box_coords': list(box_coords[kix]) + kz, 'box_score': box_scores[kix],
                                             'box_pred_class_id': cl})
    out_patient_results_list += [box for b in in_patient_results_list for box in b if box['box_type'] == 'gt']
    return [[out_patient_results_list], pid]


# ------------------------------------------------------------------------------------------------------------------ prediction pipeline
def get_mirrored_patch_crops(patch_crops, org_img_shape):
    """patch crop coordinates under the three test-time mirrorings (y, x, y&x) — predictor.py:777-816; crops are [y1, y2, x1, x2, (z1, z2)]"""
    Y, X = org_img_shape[2], org_img_shape[3]
    flip_y = lambda c: [Y - c[1], Y - c[0]] + list(c[2:])
    flip_x = lambda c: list(c[:2]) + [X - c[3], X - c[2]] + list(c[4:])
    return [[flip_y(c) for c in patch_crops], [flip_x(c) for c in patch_crops], [flip_x(flip_y(c)) for c in patch_crops]]


class _SharedPickler(pickle.Pickler):
    """Pickles one rank's predictions for the gather to rank 0.  pickle writes an object once per identity, so rank 0's raw_pred_boxes file
    has the bytes of a single-process run only if the merged lists share objects across patients as that run's do: interned strings
    (dict keys, 'det', 'gt') and numpy's built-in dtypes.  Those go by value and _SharedUnpickler resolves them to rank 0's own objects."""

    def persistent_id(self, obj):
        # sys.intern of a fresh equal string returns the interned copy if there is one (else it interns the fresh string, not obj)
        if type(obj) is str and sys.intern((obj + ' ')[:-1]) is obj:
            return b's' + obj.encode('utf-8', 'surrogatepass')
        if isinstance(obj, np.dtype) and np.dtype(obj.str) is obj:
            return b'd' + obj.str.encode()
        return None


class _SharedUnpickler(pickle.Unpickler):
    def persistent_load(self, pid):
        value = pid[1:].decode('utf-8', 'surrogatepass')
        return sys.intern(value) if pid[:1] == b's' else np.dtype(value)


def _dumps_shared(obj):
    buf = io.BytesIO()
    _SharedPickler(buf).dump(obj)
    return buf.getvalue()


def _loads_shared(data):
    return _SharedUnpickler(io.BytesIO(data)).load()


class Predictor:
    """Patient-level prediction pipeline with the call surface of the reference's `Predictor` (predictor.py:27-284): patches are forwarded in chunks of
    `cf.batch_size` (`batch_tiling_forward`), box and segmentation outputs are moved back to patient coordinates (`spatial_tiling_forward`), test
    mode adds the three mirrored passes (`data_aug_forward`) and the temporal ensemble over the best checkpoints (`predict_test_set`), and the
    boxes are consolidated by weighted box clustering / the 2D->3D merge (device kernels, csrc/consolidate.cu).

    Differences in HOW, not in WHAT: the segmentation stitching (sum of the patch label maps in float16, overlap counts, mean) runs as torch ops
    on the model's device instead of numpy slices; the per-box patch-centre factor is the closed form exp(-(d / (0.8 p))^2 / 2) of the
    reference's `norm.pdf(...) * sqrt(2 pi) * 0.8 p`; the consolidation loops over patients on the GPU instead of a 6-process pool."""

    def __init__(self, cf, net, logger, mode):
        import os
        self.cf, self.net, self.logger, self.mode = cf, net, logger, mode
        self.rank_ix = '0'                      # rank of the loaded epoch (temporal ensembling): part of every patch id
        self.n_ens = 1                          # expected predictions per position = ensembled models x test-time mirrorings
        if mode == 'test':
            try:
                self.epoch_ranking = np.load(os.path.join(cf.fold_dir, 'epoch_ranking.npy'))[:cf.test_n_epochs]
            except Exception:
                raise RuntimeError('no epoch ranking file in fold directory. seems like you are trying to run testing without prior training...')
            self.n_ens = cf.test_n_epochs * (4 if cf.test_aug else 1)

    def _info(self, msg):
        if self.logger is not None:
            self.logger.info(msg)

    # -- predictor.py:76-119
    def predict_patient(self, batch):
        self._info('evaluating patient {} for fold {} '.format(batch['pid'], getattr(self.cf, 'fold', 0)))
        self.patched_patient = 'patch_crop_coords' in batch
        results_dict = self.data_aug_forward(batch)
        if self.mode == 'val':
            for b in range(batch['patient_bb_target'].shape[0]):
                for t in range(len(batch['patient_bb_target'][b])):
                    results_dict['boxes'][b].append({'box_coords': batch['patient_bb_target'][b][t], 'box_label': batch['patient_roi_labels'][b][t],
                                                     'box_type': 'gt'})
            if self.patched_patient:
                results_dict['boxes'] = apply_wbc_to_patient([results_dict['boxes'], 'dummy_pid', self.cf.class_dict, self.cf.wcs_iou, self.n_ens])[0]
            if self.cf.merge_2D_to_3D_preds:
                results_dict['boxes'] = merge_2D_to_3D_preds_per_patient([results_dict['boxes'], 'dummy_pid', self.cf.class_dict, self.cf.merge_3D_iou])[0]
        return results_dict

    def _net_device(self):
        try:
            return next(iter(self.net.parameters())).device
        except (StopIteration, AttributeError, TypeError):
            return torch.device('cpu')

    # -- predictor.py:122-211
    def predict_test_set(self, batch_gen, return_results=True):
        """Temporal ensemble over the ranked checkpoints, mirrored passes with cf.test_aug; writes raw_pred_boxes_list.pickle (with
        cf.hold_out_test_set raw_pred_boxes_hold_out_list.pickle) to cf.fold_dir and returns the consolidated per-patient results.

        A generator from get_test_generator(cf, logger, rank, world_size) holds one rank's shard of the test set: every rank of the default
        process group (whose size must be the generator's world_size) predicts and consolidates its own patients, and rank 0 gathers them,
        writes the file in the global patient order and returns the results; the other ranks write nothing and return None.  The file's
        bytes and the results do not depend on the world size."""
        if 'world_size' in batch_gen:
            return self._predict_test_shard(batch_gen, return_results)
        out = self._predict_raw(batch_gen)
        self._write_raw(out)
        if return_results:
            return self._consolidate(out, self.n_ens, apply_wbc=True)

    def _predict_test_shard(self, batch_gen, return_results):
        import torch.distributed as dist
        world = batch_gen['world_size']
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError('predict_test_set: the test generator is sharded over {} ranks, but no process group is initialised'.format(world))
        if dist.get_world_size() != world:
            raise RuntimeError('predict_test_set: the test generator is sharded over {} ranks, but the process group has {}'.format(
                world, dist.get_world_size()))
        out = self._predict_raw(batch_gen)
        results = self._consolidate(out, self.n_ens, apply_wbc=True) if return_results else None
        rank = dist.get_rank()
        gathered = [None] * world if rank == 0 else None
        dist.gather_object(None if rank == 0 else _dumps_shared((batch_gen['shard_positions'], out, results)), gathered, dst=0)
        if rank != 0:
            return None
        parts = [(batch_gen['shard_positions'], out, results)] + [_loads_shared(b) for b in gathered[1:]]
        n = sum(len(p[0]) for p in parts)
        raw_all, results_all = [None] * n, [None] * n
        for positions, raw, res in parts:
            for j, pos in enumerate(positions):
                if not 0 <= pos < n or raw_all[pos] is not None:
                    raise RuntimeError('predict_test_set: the ranks\' shards do not partition the test set (position {} of {})'.format(pos, n))
                raw_all[pos] = raw[j]
                if return_results:
                    results_all[pos] = res[j]
        self._write_raw(raw_all)
        if return_results:
            return results_all

    def _write_raw(self, out):
        import os
        name = 'raw_pred_boxes_hold_out_list' if self.cf.hold_out_test_set else 'raw_pred_boxes_list'
        with open(os.path.join(self.cf.fold_dir, '{}.pickle'.format(name)), 'wb') as handle:
            pickle.dump(out, handle)

    def _predict_raw(self, batch_gen):
        """[[boxes per batch element (every ensemble member's detections, then the GT boxes), pid] per patient] in batch_gen's order"""
        import os
        from collections import OrderedDict
        patients = OrderedDict()
        for rank_ix, epoch in enumerate(self.epoch_ranking):
            weight_path = os.path.join(self.cf.fold_dir, '{}_best_checkpoint'.format(epoch), 'params.pth')
            self._info('tmp ensembling over rank_ix:{} epoch:{}'.format(rank_ix, weight_path))
            self.net.load_state_dict(torch.load(weight_path, map_location=self._net_device()))
            self.net.eval()
            self.rank_ix = str(rank_ix)
            with torch.no_grad():
                for _ in range(batch_gen['n_test']):
                    batch = next(batch_gen['test'])
                    if rank_ix == 0:
                        patients[batch['pid']] = {'results_list': [], 'patient_bb_target': batch['patient_bb_target'],
                                                  'patient_roi_labels': batch['patient_roi_labels']}
                    patients[batch['pid']]['results_list'].append(self.predict_patient(batch)['boxes'])
        self._info('finished predicting test set. starting post-processing of predictions.')
        out = []
        for pid, p in patients.items():
            runs = p['results_list']
            boxes = [[item for d in runs for item in d[b]] for b in range(len(runs[0]))]       # flatten the temporal ensemble per batch element
            for b in range(p['patient_bb_target'].shape[0]):
                for t in range(len(p['patient_bb_target'][b])):
                    boxes[b].append({'box_coords': p['patient_bb_target'][b][t], 'box_label': p['patient_roi_labels'][b][t], 'box_type': 'gt'})
            out.append([boxes, pid])
        return out

    # -- predictor.py:214-284
    def load_saved_predictions(self, apply_wbc=False):
        import os
        import pickle
        da = 4 if self.cf.test_aug else 1
        if not self.cf.hold_out_test_set:
            with open(os.path.join(self.cf.fold_dir, 'raw_pred_boxes_list.pickle'), 'rb') as handle:
                results = pickle.load(handle)
            n_ens = self.cf.test_n_epochs * da
        else:
            per_fold, pids = [], None
            for fold in self.cf.folds:
                with open(os.path.join(self.cf.exp_dir, 'fold_{}'.format(fold), 'raw_pred_boxes_hold_out_list.pickle'), 'rb') as handle:
                    fold_list = pickle.load(handle)
                pids = [ii[1] for ii in fold_list]
                per_fold.append([ii[0] for ii in fold_list])
            results = [[[[box for fl in per_fold for box in fl[pix][0] if box['box_type'] == 'det']], pid] for pix, pid in enumerate(pids)]
            n_ens = self.cf.test_n_epochs * da * len(self.cf.folds)
        self._info('loaded raw test set predictions with n_patients = {} and n_ens = {}'.format(len(results), n_ens))
        return self._consolidate(results, n_ens, apply_wbc)

    def _consolidate(self, results, n_ens, apply_wbc):
        if apply_wbc:
            self._info('applying wcs to test set predictions with iou = {} and n_ens = {}.'.format(self.cf.wcs_iou, n_ens))
            results = [apply_wbc_to_patient([ii[0], ii[1], self.cf.class_dict, self.cf.wcs_iou, n_ens]) for ii in results]
        if self.cf.merge_2D_to_3D_preds:
            self._info('applying 2Dto3D merging to test set predictions with iou = {}.'.format(self.cf.merge_3D_iou))
            results = [merge_2D_to_3D_preds_per_patient([ii[0], ii[1], self.cf.class_dict, self.cf.merge_3D_iou]) for ii in results]
        return results

    # -- predictor.py:278-367
    def data_aug_forward(self, batch):
        patch_crops = batch['patch_crop_coords'] if self.patched_patient else None
        results_list = [self.spatial_tiling_forward(batch, patch_crops)]
        shp = batch['original_img_shape']
        if self.mode == 'test' and self.cf.test_aug:
            mirrored = get_mirrored_patch_crops(patch_crops, shp) if self.patched_patient else [None] * 3
            img = np.copy(batch['data'])
            for n_aug, axes in enumerate([(2,), (3,), (2, 3)]):
                data = img
                for ax in axes:
                    data = np.flip(data, axis=ax)
                batch['data'] = data.copy()
                chunk = self.spatial_tiling_forward(batch, mirrored[n_aug], n_aug=str(n_aug + 1))
                for boxes in chunk['boxes']:                                   # mirror the box coordinates back
                    for box in boxes:
                        c = box['box_coords'].copy()
                        if 2 in axes:
                            c[0], c[2] = shp[2] - box['box_coords'][2], shp[2] - box['box_coords'][0]
                        if 3 in axes:
                            c[1], c[3] = shp[3] - box['box_coords'][3], shp[3] - box['box_coords'][1]
                        assert c[2] >= c[0] and c[3] >= c[1], [c, box['box_coords']]
                        box['box_coords'] = c
                seg = chunk['seg_preds']
                for ax in axes:
                    seg = np.flip(seg, axis=ax)
                chunk['seg_preds'] = seg.copy() if len(axes) == 2 else seg
                results_list.append(chunk)
            batch['data'] = img
        results_dict = {'boxes': [[item for d in results_list for item in d['boxes'][b]] for b in range(shp[0])],
                        'seg_preds': np.array([[item for d in results_list for item in d['seg_preds'][b]] for b in range(shp[0])])}
        if self.mode == 'val':
            results_dict['monitor_values'] = results_list[0]['monitor_values']
        return results_dict

    # -- predictor.py:370-455
    def spatial_tiling_forward(self, batch, patch_crops=None, n_aug='0'):
        cf = self.cf
        if patch_crops is None:
            results_dict = self.batch_tiling_forward(batch)
            for b in results_dict['boxes']:
                for box in b:
                    box['box_patch_center_factor'] = 1
                    box['box_n_overlaps'] = 1
                    box['patch_id'] = self.rank_ix + '_' + n_aug
            return results_dict
        patches = self.batch_tiling_forward(batch)
        shp = tuple(batch['original_img_shape'])
        results_dict = {'boxes': [[] for _ in range(shp[0])]}
        dev = self._net_device()
        # segmentation: sum of the patch label maps in float16 + overlap counts, then the mean where at least one patch contributes
        seg = torch.zeros((shp[0], 1) + shp[2:], dtype=torch.float16, device=dev)
        cnt = torch.zeros_like(seg, dtype=torch.uint8)
        seg_patches = torch.from_numpy(np.ascontiguousarray(patches['seg_preds'])).to(dev)
        for pix, pc in enumerate(patch_crops):
            if cf.dim == 3:
                sl = (slice(None), slice(None), slice(pc[0], pc[1]), slice(pc[2], pc[3]), slice(pc[4], pc[5]))
                seg[sl] += seg_patches[pix][None].to(torch.float16)
            else:
                sl = (slice(pc[4], pc[5]), slice(None), slice(pc[0], pc[1]), slice(pc[2], pc[3]))
                seg[sl] += seg_patches[pix].to(torch.float16)
            cnt[sl] += 1
        hit = cnt > 0
        seg[hit] = seg[hit] / cnt[hit].to(torch.float16)
        results_dict['seg_preds'] = seg.cpu().numpy()
        overlap = cnt.cpu().numpy()
        half = np.array(cf.patch_size) / 2
        for pix, pc in enumerate(patch_crops):
            for box in patches['boxes'][pix]:
                box['patch_id'] = self.rank_ix + '_' + n_aug + '_' + str(pix)
                c = box['box_coords']
                centres = [(c[ii] + c[ii + 2]) / 2 for ii in range(2)] + ([(c[4] + c[5]) / 2] if cf.dim == 3 else [])
                # boxes near the patch border are less reliable: weight = mean over the axes of a Gaussian of the centre offset (sigma = 0.8 * half size)
                box['box_patch_center_factor'] = np.mean([np.exp(-0.5 * ((bc - p) / (p * 0.8)) ** 2) for bc, p in zip(centres, half)])
                if cf.dim == 3:
                    c += np.array([pc[0], pc[2], pc[0], pc[2], pc[4], pc[4]])
                    ic = [int(np.floor(v)) if i % 2 == 0 else int(np.ceil(v)) for i, v in enumerate(c)]
                    box['box_n_overlaps'] = np.mean(overlap[:, :, ic[1]:ic[3], ic[0]:ic[2], ic[4]:ic[5]])      # index order as in predictor.py:437
                    results_dict['boxes'][0].append(box)
                else:
                    c += np.array([pc[0], pc[2], pc[0], pc[2]])
                    ic = [int(np.floor(v)) if i % 2 == 0 else int(np.ceil(v)) for i, v in enumerate(c)]
                    box['box_n_overlaps'] = np.mean(overlap[pc[4], :, ic[1]:ic[3], ic[0]:ic[2]])
                    results_dict['boxes'][pc[4]].append(box)
        if self.mode == 'val':
            results_dict['monitor_values'] = patches['monitor_values']
        return results_dict

    # -- predictor.py:458-510
    def batch_tiling_forward(self, batch):
        self._info('forwarding (patched) patient with shape: {}'.format(batch['data'].shape))
        n, bs = batch['data'].shape[0], self.cf.batch_size

        def run(b):
            if self.mode == 'val':
                return self.net.train_forward(b, is_validation=True)
            return self.net.test_forward(b, return_masks=self.cf.return_masks_in_test)

        only_det = lambda boxes: [[box for box in b if box['box_type'] == 'det'] for b in boxes]
        if n <= bs:
            results_dict = run(batch)
            if self.mode == 'val':
                results_dict['boxes'] = only_det(results_dict['boxes'])        # discard returned ground-truth / training-info boxes
            return results_dict
        chunks = []
        for start in range(0, n, bs):
            ixs = np.arange(start, min(n, start + bs))
            chunks.append(run({k: v[ixs] for k, v in batch.items() if isinstance(v, np.ndarray) and v.shape[0] == n}))
        results_dict = {'boxes': [item for d in chunks for item in d['boxes']],
                        'seg_preds': np.array([item for d in chunks for item in d['seg_preds']])}
        if self.mode == 'val':
            results_dict['monitor_values'] = {k: np.mean([d['monitor_values'][k] for d in chunks]) for k in chunks[0]['monitor_values'].keys()}
            results_dict['boxes'] = only_det(results_dict['boxes'])
        return results_dict
