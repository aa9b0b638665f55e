"""The experiments' data loader (experiments/{lidc_exp,toy_exp,pet_ct_tnm_classification}/data_loader.py with utils/dataloader_utils.py of
the reference) on this library: get_train_generators / get_test_generator with the reference's call surface, so that an exec.py-style train /
validate / test loop only swaps an import.

Training batches: BatchGenerator samples patients, 2D slices and pre-crop windows with the reference's random draws, in the reference's
order, from np.random.RandomState([seed, rank]).  Given the same draws, a run yields exactly the batches of the reference's single-worker
generator after np.random.seed([seed, rank]); 'train' and 'val_sampling' then feed the batch to augment.Augmenter, which draws from the same
stream, as the reference's transforms draw from the worker's global one.  The multi-worker order of MultiThreadedAugmenter is not reproduced
(cf.n_workers is not read).  The whole-volume scans of the reference (np.sum, np.unique, np.argwhere of the seg) read a foreground index the
device builds once per patient (csrc/loader.cu mdt_loader_fg_index); the window crop, zero padding, np.take wrap-around, slice choice and
context channels are one batched gather (mdt_loader_gather) from the in-bounds windows, which the host copies from the memory-mapped files
into a pinned staging buffer.  'data' and 'seg' of a training batch are CUDA tensors in the reference's dtypes.

Test batches: PatientBatchIterator uploads each patient once, edge-pads and tiles it into patches with one gather per output, and converts
the segs to boxes with augment.seg_to_boxes (pet_ct_tnm_classification: their connected components with augment.seg_rois); its batches are host numpy arrays in the reference's format (Predictor.predict_test_set takes
them unchanged).  The box conversion gives 'bb_target', 'roi_labels' and the relabelled 'seg' (no 'roi_masks': the predictor does not read
them).

The reference was written for numpy < 1.24, where np.array of a ragged list (class targets or boxes of patients with different ROI counts)
made an object array; this loader builds that object array where numpy >= 1.24 would raise."""
import os
from collections import OrderedDict

import numpy as np
import torch

from . import _lib as L
from . import augment as A

PETCT = 'pet_ct_tnm_classification'
SRC_DTYPE = {np.dtype(np.uint8): 0, np.dtype(np.float16): 1, np.dtype(np.float32): 2, np.dtype(np.float64): 3}
SRC_DESC = np.dtype([('offset', '<i8'), ('c', '<i4'), ('z', '<i4'), ('y', '<i4'), ('x', '<i4')])   # struct mdt_loader_src


def as_array(items):
    """np.array(items), or the 1-D object array numpy < 1.24 made of a ragged list"""
    try:
        return np.array(items)
    except ValueError:
        out = np.empty(len(items), dtype=object)
        for i, v in enumerate(items):
            out[i] = v
        return out


# ------------------------------------------------------------------------------------------------------------------- dataloader_utils
def get_class_balanced_patients(class_targets, batch_size, num_classes, slack_factor=0.1, rs=None):
    """indices of batch_size patients: the first int(batch_size * slack_factor) drawn freely, every later one redrawn until it has an ROI of the
    class rarest in the batch so far and its own rarest class is another one.  One rs.choice(len(class_targets), 1) per candidate; rs defaults
    to the global np.random."""
    rs = np.random if rs is None else rs
    picked = []
    totals = np.zeros(num_classes, dtype=np.int64)
    rarest = 0
    for ix in range(batch_size):
        while True:
            cand = rs.choice(len(class_targets), 1)[0]
            own = [class_targets[cand].count(k) for k in range(num_classes)]
            if ix < int(batch_size * slack_factor) or (np.argmin(own) != rarest and own[rarest] > 0):
                break
        totals += [class_targets[cand].count(k) for k in range(num_classes)]
        rarest = np.argmin(totals)
        picked.append(cand)
    return picked


class fold_generator:
    """cross-validation splits: get_fold_names() -> n_splits entries [train, val, test, fold] of indices into a dataset of len_data elements,
    shuffled by np.random.RandomState(seed).  The test split of fold f is the validation split of fold f - 1; split lengths are
    ceil(len_data / n_splits), one shorter in the first n_splits - len_data % n_splits folds (when len_data % n_splits > 0), and with
    len_data % n_splits == 1 the last fold's validation split hands its last element to the test split."""

    def __init__(self, seed, n_splits, len_data):
        self.myseed = seed
        self.n_splits = n_splits
        self.len_data = len_data

    def get_fold_names(self):
        names = np.arange(self.len_data)
        np.random.RandomState(self.myseed).shuffle(names)
        k = self.n_splits
        split = int(np.ceil(self.len_data / float(k)))
        mod = self.len_data % k
        short_folds = k - mod if mod > 0 else 0
        pos = list(range(self.len_data))
        te, val, tr = pos[:split], pos[split:2 * split], pos[2 * split:]
        out = []
        for fold in range(k):
            out.append([names[tr], names[val], names[te], fold])
            n_val = split - 1 if fold < short_folds else split
            leaving = list(te)
            if fold == k - 2 and mod == 1:
                leaving += val[-1:]
                val = val[:-1]
            te, val, tr = val, tr[:n_val], tr[n_val:] + leaving
        return out


def get_patch_crop_coords(img, patch_size, min_overlap=30):
    """[n_patches, 2 * dim] int crop coordinates (y0, y1, x0, x1(, z0, z1)) tiling img (y, x(, z)) with patches of patch_size: per axis
    ceil(S / P) patches (one more when neighbours would overlap by less than min_overlap) with centres np.round-ed at even spacing from P / 2
    to S - P / 2.  patch_size[2] == 1: one patch per z slice."""
    per_axis = []
    for d, s in enumerate(img.shape):
        p = patch_size[d]
        n = int(np.ceil(s / p))
        if n == 1:
            per_axis.append([(0, s)])
            continue
        step = (s - p) / (n - 1)
        if p - step < min_overlap:
            n += 1
            step = (s - p) / (n - 1)
        centres = np.round([p / 2 + step * i for i in range(n)])
        per_axis.append([(c - p / 2, c + p / 2) for c in centres])
    rows = []
    for y in per_axis[0]:
        for x in per_axis[1]:
            if len(per_axis) == 3 and patch_size[2] > 1:
                rows += [[y[0], y[1], x[0], x[1], z[0], z[1]] for z in per_axis[2]]
            elif len(per_axis) == 3 and patch_size[2] == 1:
                rows += [[y[0], y[1], x[0], x[1], z, z + 1] for z in range(img.shape[2])]
            else:
                rows.append([y[0], y[1], x[0], x[1]])
    return np.array(rows).astype(int)


def pad_nd_image(image, new_shape=None, mode="edge", kwargs=None, return_slicer=False, shape_must_be_divisible_by=None):
    """np.pad of the last len(new_shape) axes of image up to at least new_shape (never cropping), half below (rounded down) and the rest
    above; shape_must_be_divisible_by rounds each padded axis up to a multiple (an axis already a multiple grows by one multiple).  With
    return_slicer, also the slices that cut the original image back out."""
    kwargs = {} if kwargs is None else kwargs
    if new_shape is None:
        assert shape_must_be_divisible_by is not None and isinstance(shape_must_be_divisible_by, (list, tuple, np.ndarray))
        new_shape = image.shape[-len(shape_must_be_divisible_by):]
    nd = len(new_shape)
    old = np.array(image.shape[-nd:])
    target = np.array([max(new_shape[i], old[i]) for i in range(nd)])
    if shape_must_be_divisible_by is not None:
        div = shape_must_be_divisible_by
        if not isinstance(div, (list, tuple, np.ndarray)):
            div = [div] * nd
        assert len(div) == nd
        target = np.array([t - div[i] if t % div[i] == 0 else t for i, t in enumerate(target)])
        target = np.array([t + div[i] - t % div[i] for i, t in enumerate(target)])
    diff = target - old
    pads = [[0, 0]] * (len(image.shape) - nd) + [[int(d // 2), int(d // 2 + d % 2)] for d in diff]
    res = np.pad(image, pads, mode, **kwargs)
    if not return_slicer:
        return res
    pads = np.array(pads)
    pads[:, 1] = np.array(res.shape) - pads[:, 1]
    return res, [slice(*p) for p in pads]


# ------------------------------------------------------------------------------------------------------------------- dataset
def load_dataset(cf, logger, subset_ixs=None, pp_data_path=None, pp_name=None):
    """OrderedDict pid -> {'data', 'seg' (file paths), 'pid', 'class_target' (, 'fg_slices')} from the preprocessed directory's
    cf.input_df_name, as the experiment's loader builds it (cf.experiment: lidc_exp binarises malignancy scores >= 3, toy_exp reads
    'class_id' and one {pid}.npy per patient, pet_ct_tnm_classification keeps 'class_target' as it is)."""
    import pandas as pd
    if cf.server_env:
        raise NotImplementedError("server_env (copying and unpacking the dataset to a node-local directory) is not supported")
    exp = getattr(cf, 'experiment', 'lidc_exp')
    pp_data_path = cf.pp_data_path if pp_data_path is None else pp_data_path
    p_df = pd.read_pickle(os.path.join(pp_data_path, cf.input_df_name))
    if exp != 'toy_exp' and cf.select_prototype_subset is not None:
        p_df = p_df[p_df.pid.isin(p_df.pid.tolist()[:cf.select_prototype_subset])]
        logger.warning('WARNING: using prototyping data subset!!!')
    if subset_ixs is not None:
        pids_sorted = np.unique(p_df.pid.tolist())
        p_df = p_df[p_df.pid.isin([pids_sorted[ix] for ix in subset_ixs])]
        logger.info('subset: selected {} instances from df'.format(len(p_df)))
    pids = p_df.pid.tolist()
    data = OrderedDict()
    if exp == 'toy_exp':
        for pid, cid in zip(pids, p_df['class_id'].tolist()):
            path = os.path.join(pp_data_path, '{}.npy'.format(pid))
            data[pid] = {'data': path, 'seg': path, 'pid': pid, 'class_target': [cid]}
        return data
    for pid, ct, fg in zip(pids, p_df['class_target'].tolist(), p_df['fg_slices'].tolist()):
        if exp == 'lidc_exp':
            ct = [1 if c >= 3 else 0 for c in ct]
        data[pid] = {'data': os.path.join(pp_data_path, '{}_img.npy'.format(pid)), 'seg': os.path.join(pp_data_path, '{}_rois.npy'.format(pid)),
                     'pid': pid, 'class_target': ct, 'fg_slices': fg}
    return data


# ------------------------------------------------------------------------------------------------------------------- device ops
class CudaOps(object):
    """the loader's two device ops (foreground index, batched gather) and the seg-to-box conversion, on one CUDA device.  Host sources go
    through a pinned staging buffer per key, reused once the copy out of it has finished."""

    def __init__(self, device=None):
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self._staging = {}

    def _h2d(self, key, parts, dtype):
        """the flat concatenation of the host arrays `parts`, copied into the pinned buffer `key` and on to the device"""
        n = sum(int(p.size) for p in parts)
        ent = self._staging.get(key)
        if ent is None or ent[0].dtype != dtype or ent[0].size < n:
            buf = torch.empty(max(n, 1) * 3 // 2 + 1, dtype=torch.from_numpy(np.empty(0, dtype)).dtype, pin_memory=True)
            ent = (buf.numpy(), buf, torch.cuda.Event())
            ent[2].record()
            self._staging[key] = ent
        host, buf, ev = ent
        ev.synchronize()
        off = 0
        for p in parts:
            host[off:off + p.size].reshape(p.shape)[...] = p
            off += p.size
        dev = buf[:n].to(self.device, non_blocking=True)
        ev.record()
        return dev

    def fg_index(self, seg):
        """seg [Z, Y, X] uint8 -> (counts [256] int64, order [n_fg] int64) as mdt_loader_fg_index defines them"""
        Z, Y, X = seg.shape
        with torch.cuda.device(self.device):
            s = torch.from_numpy(np.array(seg, order='C')).to(self.device)
            lib = L.load()
            ws = torch.empty(lib.mdt_loader_fg_index_workspace_bytes(Z, Y, X), dtype=torch.uint8, device=self.device)
            counts = torch.empty(256, dtype=torch.int32, device=self.device)
            order = torch.empty(Z * Y * X, dtype=torch.int32, device=self.device)
            L.check(lib.mdt_loader_fg_index(L.ptr(s), Z, Y, X, L.ptr(counts), L.ptr(order), order.numel(), L.ptr(ws), ws.numel(), L.stream_ptr()))
            counts = counts.cpu().numpy().astype(np.int64)
            n_fg = int(Z * Y * X - counts[0])
            return counts, order[:n_fg].cpu().numpy().astype(np.int64)

    def upload(self, arr):
        """a whole patient array, resident on the device for the gathers of its test batches"""
        return torch.from_numpy(np.array(arr, order='C')).to(self.device)

    def gather(self, src, elems, tabs, out_dtype, key='src'):
        """out [n, C, I, J, K] = mdt_loader_gather of src (a device tensor from upload, or a list of host windows staged under `key`, one
        per element, elems[b].offset then into their concatenation), tabs = (tab_c [n, C], tab_z [n, C, K], tab_y [n, I], tab_x [n, J])"""
        tab_c, tab_z, tab_y, tab_x = tabs
        n, C = tab_c.shape
        I, J, K = tab_y.shape[1], tab_x.shape[1], tab_z.shape[2]
        with torch.cuda.device(self.device):
            if isinstance(src, list):
                dt = src[0].dtype
                src = self._h2d(key, src, dt)
            else:
                dt = np.dtype(str(src.dtype).replace('torch.', ''))
            if dt not in SRC_DTYPE:
                raise ValueError("unsupported source dtype %s" % dt)
            meta = np.concatenate([elems.view(np.int32).reshape(-1), tab_c.reshape(-1), tab_z.reshape(-1), tab_y.reshape(-1), tab_x.reshape(-1)])
            meta = self._h2d(key + '_tabs', [meta.astype(np.int32)], np.dtype(np.int32))
            ptr = lambda k: ctypes_ptr(meta, k)
            offs = np.cumsum([6 * n, n * C, n * C * K, n * I])     # tab_c, tab_z, tab_y, tab_x after the element descriptors
            out = torch.empty((n, C, I, J, K), dtype=torch.from_numpy(np.empty(0, out_dtype)).dtype, device=self.device)
            L.check(L.load().mdt_loader_gather(SRC_DTYPE[dt], L.ptr(src), ptr(0), n, C, I, J, K, ptr(offs[0]), ptr(offs[1]), ptr(offs[2]), ptr(offs[3]),
                                               SRC_DTYPE[np.dtype(out_dtype)], L.ptr(out), L.stream_ptr()))
            return out

    def seg_rois(self, seg, class_target, class_specific):
        """seg [B, 1, *P] device uint8, class_target [B] host int32 -> (elem_first [B + 1] host int32, stats [elem_first[B], 7] host int32,
        relabelled seg on the device) of augment.seg_rois"""
        with torch.cuda.device(self.device):
            ct = torch.from_numpy(np.ascontiguousarray(class_target, dtype=np.int32)).to(self.device)
            _, first, stats, seg_out = A.seg_rois(seg.contiguous(), ct, class_specific)
            first = first.cpu().numpy()
            return first, stats[:int(first[-1])].cpu().numpy(), seg_out

    def seg_to_boxes(self, seg, lut):
        """seg [B, 1, *P] device uint8, lut [B, 256] host uint8 -> (stats [B, 255, 7] host int32, relabelled seg on the device)"""
        with torch.cuda.device(self.device):
            stats, seg_out, _ = A.seg_to_boxes(seg.contiguous(), torch.from_numpy(lut).to(self.device))
            return stats.cpu().numpy(), seg_out

    def to_host(self, t):
        return t.cpu().numpy()


def ctypes_ptr(t, elem_offset):
    import ctypes
    return ctypes.c_void_p(t.data_ptr() + 4 * int(elem_offset))


# ------------------------------------------------------------------------------------------------------------------- foreground index
class FgIndex(object):
    """one patient's foreground on the host: counts [256] per label and order [n_fg], the (y, x, z) linear indices grouped by label, each
    group in np.argwhere order of the transposed (y, x, z) seg"""

    def __init__(self, counts, order, shape):
        self.counts = np.asarray(counts, dtype=np.int64)
        self.order = np.asarray(order, dtype=np.int64)
        self.shape = tuple(int(s) for s in shape)          # (Y, X, Z)
        self.ends = np.cumsum(self.counts[1:])
        self._slice_counts = None

    def group(self, label):
        return self.order[(self.ends[label - 2] if label > 1 else 0):self.ends[label - 1]]

    def labels_of_order(self):
        return np.repeat(np.arange(1, 256), self.counts[1:])

    def slice_counts(self):
        """[Z, 256] foreground voxels per (z slice, label); built on first use from the index"""
        if self._slice_counts is None:
            Z = self.shape[2]
            self._slice_counts = np.bincount((self.order % Z) * 256 + self.labels_of_order(), minlength=Z * 256).reshape(Z, 256)
        return self._slice_counts

    def coords(self, idx, slice_id=None):
        Y, X, Z = self.shape
        c = [idx // (X * Z), (idx // Z) % X, idx % Z]
        return np.stack(c[:2] if slice_id is not None else c, axis=1)


class _View(object):
    """the seg the reference's BatchGenerator scans: the transposed patient volume, or one of its z slices (slice_id), zero-padded by
    `below` voxels at the start of each axis to `shape`"""

    def __init__(self, index, slice_id, below, shape):
        self.ix, self.slice_id, self.below, self.shape = index, slice_id, np.asarray(below, dtype=np.int64), shape

    def _label_counts(self):
        return self.ix.counts if self.slice_id is None else self.ix.slice_counts()[self.slice_id]

    def any_fg(self):
        return int(self._label_counts()[1:].sum()) > 0

    def unique(self):
        """np.unique of the padded view"""
        c = self._label_counts()
        bg = int(np.prod(self.shape)) - int(c[1:].sum())
        return np.array(([0] if bg > 0 else []) + [int(l) for l in np.nonzero(c[1:])[0] + 1], dtype=np.uint8)

    def _select(self, idx):
        if self.slice_id is not None:
            idx = idx[idx % self.ix.shape[2] == self.slice_id]
        return self.ix.coords(idx, self.slice_id) + self.below

    def argwhere(self, label):
        return self._select(self.ix.group(int(label)))

    def any_fg_in(self, windows):
        """any foreground voxel inside the per-axis windows {axis: (min_crop, max_crop)} (np.take: negative indices wrap)"""
        c = self._select(self.ix.order)
        inside = np.ones(len(c), dtype=bool)
        for ax, (lo, hi) in windows.items():
            inside &= ((c[:, ax] - lo) % self.shape[ax]) < (hi - lo)
        return bool(inside.any())


def _window(tables):
    """(lo, hi) bounding the valid (>= 0) entries of an index table, and the table made relative to lo"""
    t = np.asarray(tables)
    v = t[t >= 0]
    if v.size == 0:
        return (0, 1), np.full(t.shape, -1, dtype=np.int32)
    lo, hi = int(v.min()), int(v.max()) + 1
    return (lo, hi), np.where(t >= 0, t - lo, -1).astype(np.int32)


def _src_desc(shapes):
    d = np.zeros(len(shapes), dtype=SRC_DESC)
    off = 0
    for b, s in enumerate(shapes):
        d[b] = (off, *s)
        off += int(np.prod(s))
    return d


# ------------------------------------------------------------------------------------------------------------------- BatchGenerator
class BatchGenerator(object):
    """pre-crop training batches of the experiment's BatchGenerator.generate_train_batch (cf.experiment selects lidc_exp, toy_exp or
    pet_ct_tnm_classification), drawn from np.random.RandomState([seed, rank]) (rank: the torch.distributed rank, else 0).  ops: the device
    ops (CudaOps on the current device by default).  Batches: 'data' [B, C, *pre_crop] and 'seg' [B, 1, *pre_crop] uint8 as the ops
    return them (CUDA tensors), 'pid' list, 'class_target'."""

    def __init__(self, data, batch_size, cf, seed=0, rank=None, ops=None):
        if rank is None:
            import torch.distributed as dist
            rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        self._data = data
        self.batch_size = batch_size
        self.cf = cf
        self.exp = getattr(cf, 'experiment', 'lidc_exp')
        self.rs = np.random.RandomState([int(seed), int(rank)])
        self.ops = ops if ops is not None else CudaOps()
        self.crop_margin = np.array(cf.patch_size) / 8.
        self.p_fg = 0.5
        self._index = {}

    def __iter__(self):
        return self

    def __next__(self):
        return self.generate_train_batch()

    def fg_index(self, pid, seg):
        """the patient's FgIndex, built on the device on first use and cached"""
        ix = self._index.get(pid)
        if ix is None:
            if seg.dtype != np.uint8:
                raise ValueError("patient %s: seg files must be uint8 instance maps, got %s" % (pid, seg.dtype))
            counts, order = self.ops.fg_index(seg)
            ix = self._index[pid] = FgIndex(counts, order, (seg.shape[1], seg.shape[2], seg.shape[0]))
        return ix

    def generate_train_batch(self):
        cf, rs = self.cf, self.rs
        patients = list(self._data.items())
        targets_list = [v['class_target'] for (k, v) in patients]
        if self.exp == PETCT:
            batch_ixs = rs.choice(len(targets_list), self.batch_size)
        elif self.exp == 'toy_exp' or cf.head_classes > 2:
            batch_ixs = get_class_balanced_patients(targets_list, self.batch_size, cf.head_classes - 1, slack_factor=cf.batch_sample_slack, rs=rs)
        else:
            batch_ixs = rs.choice(len(targets_list), self.batch_size)
        if self.exp == 'toy_exp':
            return self._toy_batch([patients[b][1] for b in batch_ixs])
        plans = [self._plan(patients[b][1]) for b in batch_ixs]
        pids = [str(p['pid']) if self.exp == PETCT else p['pid'] for p in (patients[b][1] for b in batch_ixs)]
        targets = [pl['class_target'] for pl in plans]
        out_dtype = np.float16 if self.exp == PETCT else plans[0]['dtype']
        data = self._gather(plans, 'data', out_dtype)
        seg = self._gather(plans, 'seg', np.uint8)
        return {'data': data, 'seg': seg, 'pid': pids, 'class_target': targets if self.exp == PETCT else as_array(targets)}

    def _toy_batch(self, patients):
        files = [np.load(p['data'], mmap_mode='r') for p in patients]
        _, Y, X = files[0].shape
        n = len(files)
        tabs = lambda ch: (np.full((n, 1), ch, np.int32), np.zeros((n, 1, 1), np.int32), np.tile(np.arange(Y, dtype=np.int32), (n, 1)),
                           np.tile(np.arange(X, dtype=np.int32), (n, 1)))
        windows = [np.asarray(f)[:, None] for f in files]
        elems = _src_desc([w.shape for w in windows])
        data = self.ops.gather(windows, elems, tabs(0), files[0].dtype, key='data')[..., 0]
        seg = self.ops.gather(windows, elems, tabs(1), np.uint8, key='seg')[..., 0]
        return {'data': data, 'seg': seg, 'pid': [p['pid'] for p in patients], 'class_target': as_array([p['class_target'] for p in patients])}

    def _plan(self, patient):
        """one element: the random draws and the index tables of its pre-crop window"""
        cf, rs = self.cf, self.rs
        img = np.load(patient['data'], mmap_mode='r')
        seg = np.load(patient['seg'], mmap_mode='r')
        if img.ndim == 3:
            img = img[None]
        C, Z, Y, X = img.shape
        index = self.fg_index(patient['pid'], seg)
        slice_id = None
        if cf.dim == 2:
            fg = patient['fg_slices']
            if len(fg) > 0:
                fg_prob = self.p_fg / len(fg)
                bg_prob = (1 - self.p_fg) / (Z - len(fg))
                slice_id = rs.choice(Z, p=[fg_prob if ix in fg else bg_prob for ix in range(Z)])
            else:
                slice_id = rs.choice(Z)
            n = cf.n_3D_context
            if n is not None:
                tab_c = np.zeros(2 * n + 1, np.int64)
                tab_z = np.array([[z if 0 <= z < Z else -1] for z in range(slice_id - n, slice_id + n + 1)])
            else:
                tab_c = np.arange(C)
                tab_z = np.full((C, 1), slice_id)
            axes = [np.arange(Y), np.arange(X)]
            seg_z = np.array([[slice_id]])
        else:
            tab_c = np.arange(C)
            axes = [np.arange(Y), np.arange(X), np.arange(Z)]
        pre = cf.pre_crop_size
        shape = [len(a) for a in axes]
        below = [0] * len(axes)
        if any(shape[d] < ps for d, ps in enumerate(pre)):
            for d, ps in enumerate(pre):
                diff = max(shape[d], ps) - shape[d]
                below[d] = diff // 2
                axes[d] = np.concatenate([np.full(diff // 2, -1), axes[d], np.full(diff - diff // 2, -1)])
            shape = [len(a) for a in axes]
        view = _View(index, slice_id, below, shape)
        crop_dims = [d for d, ps in enumerate(pre) if shape[d] > ps]
        windows = {}
        if len(crop_dims) > 0:
            fg_prob_sample = rs.rand(1)
            if fg_prob_sample < self.p_fg and view.any_fg():
                seg_ixs = view.argwhere(rs.choice(view.unique()[1:], 1)[0])
                anchor = seg_ixs[rs.choice(seg_ixs.shape[0], 1)][0]
                centre = {}
                for ii in crop_dims:
                    low = np.max((pre[ii] // 2, anchor[ii] - (cf.patch_size[ii] // 2 - self.crop_margin[ii])))
                    high = np.min((shape[ii] - pre[ii] // 2, anchor[ii] + (cf.patch_size[ii] // 2 - self.crop_margin[ii])))
                    if low >= high:
                        wide = 1 if self.exp == PETCT else 0
                        low = shape[ii] // 2 - (shape[ii] // 2 - pre[ii] // 2) - wide
                        high = shape[ii] // 2 + (shape[ii] // 2 - pre[ii] // 2) + wide
                    centre[ii] = rs.randint(low=low, high=high)
            else:
                centre = {ii: rs.randint(low=pre[ii] // 2, high=shape[ii] - pre[ii] // 2) for ii in crop_dims}
            for ii in crop_dims:
                lo, hi = int(centre[ii] - pre[ii] // 2), int(centre[ii] + pre[ii] // 2)
                windows[ii] = (lo, hi)
                axes[ii] = axes[ii][np.arange(lo, hi)]
        if self.exp == PETCT:
            class_target = 0 if (view.any_fg_in(windows) if windows else view.any_fg()) else -1
        else:
            class_target = patient['class_target']
        if cf.dim == 3:
            tab_z = np.tile(axes[2], (len(tab_c), 1))
            seg_z = axes[2][None]
        return {'img': img, 'seg': seg, 'tab_c': tab_c, 'tab_z': tab_z, 'seg_z': seg_z, 'y': axes[0], 'x': axes[1], 'dtype': img.dtype,
                'class_target': class_target}

    def _gather(self, plans, which, out_dtype):
        windows, tabs = [], [[], [], [], []]
        for pl in plans:
            tc, tz = (pl['tab_c'], pl['tab_z']) if which == 'data' else (np.zeros(1, np.int64), pl['seg_z'])
            (c0, c1), rc = _window(tc)
            (z0, z1), rz = _window(tz)
            (y0, y1), ry = _window(pl['y'])
            (x0, x1), rx = _window(pl['x'])
            src = pl['img'] if which == 'data' else pl['seg'][None]
            w = src[c0:c1, z0:z1, y0:y1, x0:x1]
            windows.append(w if w.dtype == plans[0]['dtype'] or which == 'seg' else w.astype(plans[0]['dtype']))
            for t, r in zip(tabs, (rc, rz, ry, rx)):
                t.append(r)
        elems = _src_desc([w.shape for w in windows])
        out = self.ops.gather(windows, elems, tuple(np.stack(t).astype(np.int32) for t in tabs), out_dtype, key=which)
        return out[..., 0] if self.cf.dim == 2 else out


# ------------------------------------------------------------------------------------------------------------------- PatientBatchIterator
def _edge(S, new):
    """index table of np.pad(mode='edge') of an axis of S voxels to new"""
    return np.clip(np.arange(new) - (new - S) // 2, 0, S - 1)


class PatientBatchIterator(object):
    """one patient per batch, as the experiment's PatientBatchIterator.generate_train_batch builds it: the patient edge-padded to at least
    cf.patch_size, its patient-level targets (3D, or per slice in 2D plus the 3D targets with merge_2D_to_3D_preds), and, when it is larger
    than a patch, all its overlapping patches ('patch_crop_coords').  Host numpy arrays in the reference's format.

    pet_ct_tnm_classification: the reference's iterator cannot run (it indexes a file listing with an integer, reads an unset dataset_pids
    and converts boxes without a seg) and preprocesses raw scans on the fly.  Here it is the lidc_exp iterator on the preprocessed two-channel
    directory (petct_preprocessing): both image channels (with n_3D_context, the CT's context slices, as BatchGenerator stacks them), the
    ROIs of the patient and of every patch taken as the connected components of the seg, and the patient's target 0 if its seg has any
    foreground, else -1 (the rule of the experiment's BatchGenerator)."""

    def __init__(self, data, cf, ops=None):
        self._data = data
        self.cf = cf
        self.exp = getattr(cf, 'experiment', 'lidc_exp')
        self.ops = ops if ops is not None else CudaOps()
        self.patient_ix = 0
        self.dataset_pids = [v['pid'] for (k, v) in data.items()]
        self.patch_size = list(cf.patch_size) + ([1] if len(cf.patch_size) == 2 else [])

    def __iter__(self):
        return self

    def __next__(self):
        return self.generate_train_batch()

    def _boxes(self, seg, class_targets, dim):
        if self.exp == PETCT:
            first, stats, seg_out = self.ops.seg_rois(seg, np.asarray(class_targets, dtype=np.int32).reshape(-1), self.cf.class_specific_seg_flag)
            bb, labels, _ = A.boxes_from_rois(first, stats, class_targets, dim)
            return as_array(bb), as_array(labels), self.ops.to_host(seg_out)
        lut = A.label_lut(class_targets, self.cf.class_specific_seg_flag)
        stats, seg_out = self.ops.seg_to_boxes(seg, lut)
        bb, labels, _ = A.boxes_from_stats(stats, class_targets, dim)
        return as_array(bb), as_array(labels), self.ops.to_host(seg_out)

    def generate_train_batch(self):
        cf = self.cf
        pid = self.dataset_pids[self.patient_ix]
        patient = self._data[pid]
        targets = np.array([patient['class_target']])
        if self.exp == 'toy_exp':
            out = self._toy(patient, pid, targets)
        else:
            out = self._lidc(patient, pid, targets)
        self.patient_ix = (self.patient_ix + 1) % len(self.dataset_pids)
        return out

    def _toy(self, patient, pid, targets):
        f = np.load(patient['data'], mmap_mode='r')
        _, Y, X = f.shape
        src = self.ops.upload(np.asarray(f)[:, None])
        desc = _src_desc([(2, 1, Y, X)])
        tabs = lambda ch: (np.array([[ch]], np.int32), np.zeros((1, 1, 1), np.int32), np.arange(Y, dtype=np.int32)[None], np.arange(X, dtype=np.int32)[None])
        data = self.ops.to_host(self.ops.gather(src, desc, tabs(0), f.dtype, key='test')[..., 0])
        seg = self.ops.gather(src, desc, tabs(1), np.uint8, key='test')[..., 0]
        bb, labels, seg = self._boxes(seg, targets, 2)
        return {'data': data, 'seg': seg, 'class_target': targets, 'pid': pid, 'bb_target': bb, 'roi_labels': labels, 'patient_bb_target': bb,
                'patient_roi_labels': labels, 'original_img_shape': data.shape}

    def _lidc(self, patient, pid, targets):
        cf = self.cf
        img = np.load(patient['data'], mmap_mode='r')
        seg_f = np.load(patient['seg'], mmap_mode='r')
        if img.ndim == 3:
            img = img[None]
        C, Z, Y, X = img.shape
        if self.exp == PETCT:
            targets = np.array([0 if np.asarray(seg_f).any() else -1])
        img_dev = self.ops.upload(img)
        seg_dev = self.ops.upload(seg_f)
        d_img, d_seg = _src_desc([(C, Z, Y, X)]), _src_desc([(1, Z, Y, X)])
        P = self.patch_size
        shape = [max(s, p) for s, p in zip((Y, X, Z), P)]
        ey, ex, ez = _edge(Y, shape[0]), _edge(X, shape[1]), _edge(Z, shape[2])
        n3 = cf.n_3D_context
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)

        def gather(src, desc, n, tz, ty, tx, dtype, chans=(0,)):
            """chans: the source channel of each output channel; tz [n or 1, C or 1, K] broadcast over them"""
            d = np.repeat(desc, n)
            tz = np.asarray(tz)
            tabs = (i32(np.tile(chans, (n, 1))), i32(np.broadcast_to(tz, (n, len(chans), tz.shape[-1]))), i32(ty), i32(tx))
            return self.ops.gather(src, d, tabs, dtype, key='test')

        def slice_z(zs, context):
            """[n, C, 1] z tables of slices zs, with the context channels (0 outside the volume) when context"""
            zs = np.asarray(zs)
            if not context:
                return zs[:, None, None]
            zz = zs[:, None] + np.arange(-n3, n3 + 1)[None]
            return np.where((zz >= 0) & (zz < Z), zz, -1)[..., None]

        chans = np.arange(C)                                   # image channels, or the CT's context slices in 2D with n_3D_context
        chans2 = np.zeros(2 * n3 + 1, np.int64) if n3 is not None else chans
        patched = any(shape[d] > P[d] for d in range(3))
        out = {}
        if cf.dim == 3 or cf.merge_2D_to_3D_preds:
            seg3 = gather(seg_dev, d_seg, 1, ez[None, None], ey[None], ex[None], np.uint8)
            bb3, lab3, seg3_out = self._boxes(seg3, targets, 3)
            shape3 = (1, 1, *shape)
            if cf.dim == 3:
                out = {'seg': seg3_out, 'class_target': targets, 'pid': pid, 'bb_target': bb3, 'roi_labels': lab3}
                if not patched:
                    out['data'] = self.ops.to_host(gather(img_dev, d_img, 1, ez[None, None], ey[None], ex[None], img.dtype, chans))
            out.update({'patient_bb_target': bb3, 'patient_roi_labels': lab3, 'original_img_shape': shape3})
        if cf.dim == 2:
            Zp = shape[2]
            zs = ez
            C2 = len(chans2)
            seg2 = gather(seg_dev, d_seg, Zp, slice_z(zs, False), np.tile(ey, (Zp, 1)), np.tile(ex, (Zp, 1)), np.uint8)[..., 0]
            targets2 = np.array(np.repeat(targets, Zp, axis=0))
            bb2, lab2, seg2_out = self._boxes(seg2, targets2, 2)
            shape2 = (Zp, C2, shape[0], shape[1])
            out_2d = {'seg': seg2_out, 'class_target': targets2, 'pid': pid, 'bb_target': bb2, 'roi_labels': lab2, 'original_img_shape': shape2}
            if not patched:
                out_2d['data'] = self.ops.to_host(gather(img_dev, d_img, Zp, slice_z(zs, n3 is not None), np.tile(ey, (Zp, 1)), np.tile(ex, (Zp, 1)),
                                                         img.dtype, chans2)[..., 0])
            if cf.merge_2D_to_3D_preds:
                out_2d.update({'patient_bb_target': out['patient_bb_target'], 'patient_roi_labels': out['patient_roi_labels']})
            else:
                out_2d.update({'patient_bb_target': bb2, 'patient_roi_labels': lab2})
            out = out_2d
        if not patched:
            return out
        coords = get_patch_crop_coords(np.broadcast_to(np.uint8(0), shape), P)
        n = len(coords)
        ty = np.stack([ey[c[0]:c[1]] for c in coords])
        tx = np.stack([ex[c[2]:c[3]] for c in coords])
        if cf.dim == 3:
            tz = np.stack([ez[c[4]:c[5]] for c in coords])[:, None]
            data = gather(img_dev, d_img, n, tz, ty, tx, img.dtype, chans)
            seg = gather(seg_dev, d_seg, n, tz, ty, tx, np.uint8)
        else:
            zs = ez[coords[:, 4]]
            data = gather(img_dev, d_img, n, slice_z(zs, n3 is not None), ty, tx, img.dtype, chans2)[..., 0]
            seg = gather(seg_dev, d_seg, n, slice_z(zs, False), ty, tx, np.uint8)[..., 0]
        targets_p = np.repeat(targets, n, axis=0)
        bb, labels, seg_out = self._boxes(seg, targets_p, cf.dim)
        return {'data': self.ops.to_host(data), 'seg': seg_out, 'class_target': targets_p, 'pid': pid, 'patch_crop_coords': np.array(coords),
                'patient_bb_target': out['patient_bb_target'], 'patient_roi_labels': out['patient_roi_labels'],
                'original_img_shape': out['original_img_shape'], 'bb_target': bb, 'roi_labels': labels}


# ------------------------------------------------------------------------------------------------------------------- pipelines
class _Augmented(object):
    """BatchGenerator -> Augmenter, both drawing from the generator's RandomState as the reference's pipeline draws from one global stream"""

    def __init__(self, gen, aug):
        self.gen, self.aug = gen, aug
        aug.rs = gen.rs

    def __iter__(self):
        return self

    def __next__(self):
        return self.aug(self.gen.generate_train_batch())


def _pipeline(data, cf, is_training, rank=None):
    gen = BatchGenerator(data, cf.batch_size, cf, seed=cf.seed, rank=rank)
    aug = A.Augmenter(cf, is_training=is_training, seed=cf.seed, rank=rank, with_masks=cf.model == 'mrcnn' and not cf.frcnn_mode,
                      get_rois_from_seg_flag=getattr(cf, 'experiment', 'lidc_exp') == PETCT)
    return _Augmented(gen, aug)


def get_train_generators(cf, logger):
    """{'train', 'val_sampling', 'val_patient' (cf.val_mode == 'val_patient'), 'n_val'}: the experiment's cross-validation split (toy_exp:
    its fixed train / val split of the first cf.n_train_val_data patients), 'train' augmented, 'val_sampling' center-cropped, each batch as
    net.train_forward takes it.  The fold pickle is written to / read from cf.exp_dir as the reference does."""
    import pickle
    all_data = load_dataset(cf, logger)
    all_pids = np.unique([v['pid'] for (k, v) in all_data.items()])
    if getattr(cf, 'experiment', 'lidc_exp') == 'toy_exp':
        assert cf.n_train_val_data <= len(all_pids), "requested {} train val samples, but dataset only has {} train val samples.".format(
            cf.n_train_val_data, len(all_pids))
        train_pids = list(all_pids[:int(2 * cf.n_train_val_data // 3)])
        val_pids = list(all_pids[int(np.ceil(2 * cf.n_train_val_data // 3)):cf.n_train_val_data])
        n_val_ix = len(val_pids)
    else:
        path = os.path.join(cf.exp_dir, 'fold_ids.pickle')
        if not cf.created_fold_id_pickle:
            fg = fold_generator(seed=cf.seed, n_splits=cf.n_cv_splits, len_data=len(all_pids)).get_fold_names()
            with open(path, 'wb') as handle:
                pickle.dump(fg, handle)
            cf.created_fold_id_pickle = True
        else:
            with open(path, 'rb') as handle:
                fg = pickle.load(handle)
        train_ix, val_ix, test_ix, _ = fg[cf.fold]
        train_pids = [all_pids[ix] for ix in train_ix]
        val_pids = [all_pids[ix] for ix in val_ix]
        if cf.hold_out_test_set:
            train_pids += [all_pids[ix] for ix in test_ix]
        n_val_ix = len(val_ix)
    train_data = OrderedDict((k, v) for (k, v) in all_data.items() if v['pid'] in set(train_pids))
    val_data = OrderedDict((k, v) for (k, v) in all_data.items() if v['pid'] in set(val_pids))
    logger.info("data set loaded with: {} train / {} val patients".format(len(train_pids), len(val_pids)))
    batch_gen = {'train': _pipeline(train_data, cf, True), 'val_sampling': _pipeline(val_data, cf, False)}
    if cf.val_mode == 'val_patient':
        batch_gen['val_patient'] = PatientBatchIterator(val_data, cf)
        batch_gen['n_val'] = n_val_ix if cf.max_val_patients is None else min(n_val_ix, cf.max_val_patients)
    else:
        batch_gen['n_val'] = cf.num_val_batches
    return batch_gen


def get_test_generator(cf, logger, rank=None, world_size=None):
    """{'test': PatientBatchIterator, 'n_test'}: the hold-out directory cf.pp_test_data_path with cf.hold_out_test_set, else the fold's test
    split of cf.exp_dir's fold pickle.

    With rank and world_size (one process per GPU): the first n_test patients (the cf.max_test_patients cap on the whole ordered list) are
    sharded round-robin, and this rank keeps positions rank, rank + world_size, ...  Its iterator reads only those patients, 'n_test' is
    their count (0 when world_size exceeds it), and 'shard_positions' (their positions in the capped list) and 'world_size' make
    Predictor.predict_test_set gather every rank's results to rank 0."""
    import operator
    import pickle
    if (rank is None) != (world_size is None):
        raise ValueError("get_test_generator: give both rank and world_size or neither (rank={}, world_size={})".format(rank, world_size))
    if world_size is not None:
        rank, world_size = operator.index(rank), operator.index(world_size)
        if not 0 <= rank < world_size:
            raise ValueError("get_test_generator: rank {} is outside [0, world_size = {})".format(rank, world_size))
    if cf.hold_out_test_set:
        test_ix = None
    else:
        with open(os.path.join(cf.exp_dir, 'fold_ids.pickle'), 'rb') as handle:
            _, _, test_ix, _ = pickle.load(handle)[cf.fold]
    test_data = load_dataset(cf, logger, test_ix, pp_data_path=cf.pp_test_data_path)
    n = len(test_data)
    logger.info("data set loaded with: {} test patients".format(n))
    n_test = n if cf.max_test_patients == "all" else min(cf.max_test_patients, n)
    if world_size is None:
        return {'test': PatientBatchIterator(test_data, cf), 'n_test': n_test}
    positions = list(range(rank, n_test, world_size))
    patients = list(test_data.items())
    logger.info("rank {} of {}: {} of the {} test patients".format(rank, world_size, len(positions), n_test))
    return {'test': PatientBatchIterator(OrderedDict(patients[p] for p in positions), cf), 'n_test': len(positions),
            'shard_positions': positions, 'world_size': world_size}
