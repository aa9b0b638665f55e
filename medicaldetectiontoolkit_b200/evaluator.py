"""Evaluator: scores detections against ground truth, with the call surface of the reference's evaluator.py (Evaluator(cf, logger, mode),
evaluate_predictions, return_metrics, score_test_df and the test_df attribute).

The matching of detections to ground truth, the ROI-level AP and the patient-level counts run as kernels of csrc/evaluate.cu; the host
flattens the box dicts into arrays in one Python pass, and afterwards does only O(rows) numpy bookkeeping and scikit-learn's few
O(#thresholds) curve expressions, so every AP, AUC and curve equals the reference's bit for bit.  There is no CPU fallback: without a CUDA
device the calls raise, like the other native ops.

Dependencies: scikit-learn is never imported.  pandas is imported only to build `test_df` (on first access) and to write or read the
per-fold `*_test_df.pickle` files, which are the reference's format; the scores themselves need only numpy.

Plots: when cf.plot_dir names an existing directory (the reference's runner creates it before training), return_metrics writes the
reference's files there with plotting.py (rendered on the GPU; matplotlib is not a dependency): with cf.plot_prediction_histograms,
pred_hist_{fold}_{val|mode}_{level}_cl{cl}.png per class and score level; with cf.plot_stat_curves, {fold}_{mode}_stat_curves_{roc|prc}.png.
Without one (no plot_dir, None, or a path that is not a directory) it writes nothing.  Documented deviation:
the reference's plot_stat_curves raises on a patient-level stat whose curve is np.nan (a class with one label value), indexing nan[0];
here that curve is skipped.

Documented deviation: with cf.scan_det_thresh the reference passes the ROI APs at the thresholds np.arange(0.9, 1, 0.01) to logger.info
as a stray argument, so they are never printed; here they are formatted into the message.  They are computed at the 'rois' score level
only: at the 'patient' level the reference's scan fails (its per-patient frame has no match_iou column).  return_metrics returns what the
reference returns.

Scores and coordinates are promoted to fp64.  Ground-truth coordinates often arrive as integer arrays; the reference computes their
volumes in int64 and mixes them with fp64, and promoting them to fp64 first gives the same values as long as coordinates and volumes stay
below 2^53.  For ROI-level ties in score, rows keep their row order (the reference's pandas quicksort leaves it undefined).

Beyond the reference: Evaluator.bootstrap / score_bootstrap give patient-bootstrap confidence intervals and the (step) FROC / CPM of the
stored rows, each resample evaluated on the device from weighted counts (see Evaluator.bootstrap for the definitions).
"""
import os

import numpy as np
import torch

from . import _lib as L
from . import plotting

TYPES = ('det_tp', 'det_fp', 'det_fn', 'patient_tn')      # type codes 0..3 of csrc/evaluate.cu
RECALL_POINTS = np.linspace(.0, 1, 101, endpoint=True)      # compute_roi_ap's R
SCAN_THRESHOLDS = list(np.arange(0.9, 1, 0.01))            # return_metrics' conf_threshs
FROC_RATES = (0.125, 0.25, 0.5, 1, 2, 4, 8)                # false positives per scan of the FROC; their mean sensitivity is the CPM
BOOTSTRAP_CHUNK_BYTES = 64 << 20                           # bound on the device outputs of one bootstrap call (resamples per call follow)
_TYPES_ARR = np.array(TYPES, dtype=object)


def _unique_in_order(a):
    """pandas' Series.unique(): the distinct values in order of first appearance, and the index of each element's value among them"""
    u, first, inv = np.unique(a, return_index=True, return_inverse=True)
    order = np.argsort(first, kind='stable')
    rank = np.empty(order.size, dtype=np.int64)
    rank[order] = np.arange(order.size)
    return u[order], rank[inv.reshape(-1)]


def _device():
    if not torch.cuda.is_available():
        raise L.MdtError("the Evaluator runs on CUDA only (there is no CPU fallback) and no CUDA device is available")
    return torch.device('cuda', torch.cuda.current_device())


class _Outputs:
    """the caller-owned outputs of one evaluation call, carved from one device buffer so that they return in one device-to-host copy"""

    def __init__(self, dev, specs):
        self.layout, off = {}, 0
        for name, dtype, count in specs:
            nbytes = np.dtype(dtype).itemsize * max(int(count), 1)
            self.layout[name] = (np.dtype(dtype), int(count), off)
            off += (nbytes + 15) // 16 * 16
        self.buf = torch.empty(max(off, 16), dtype=torch.uint8, device=dev)

    def ptr(self, name):
        return L.ctypes.c_void_p(self.buf.data_ptr() + self.layout[name][2])

    def fetch(self):
        host = self.buf.cpu().numpy()
        return {n: host[off:off + dt.itemsize * c].view(dt) for n, (dt, c, off) in self.layout.items()}


def _dev(a, dev, dtype):
    return torch.from_numpy(np.array(a, dtype=dtype)).to(dev)      # a copy: the columns may be read-only views


def _workspace(nbytes, dev):
    if nbytes == 0:
        raise L.MdtError("libmdt_b200: the evaluation workspace could not be sized")
    return torch.empty(int(nbytes), dtype=torch.uint8, device=dev)


def _scalar(v):
    return v.item() if isinstance(v, np.ndarray) and v.ndim == 0 else v


def flatten_results(batch_elements_list, classes):
    """One Python pass over the box dicts of every element: the 'det' boxes of a class in cf.class_dict and the 'gt' boxes with such a
    label (other box types, e.g. the anchor-monitoring boxes, are ignored), grouped by (element, class index) in their list order.
    Returns dim, candidate boxes / scores / offsets, GT boxes / offsets and the per-patient element offsets."""
    cidx = {cl: k for k, cl in enumerate(classes)}
    nc = len(classes)
    ck, cc, cs, gk, gc, n_elem = [], [], [], [], [], []
    e = 0
    for elements in batch_elements_list:
        n_elem.append(len(elements))
        for boxes in elements:
            base = e * nc
            for box in boxes:
                t = box['box_type']
                if t == 'det':
                    k = cidx.get(_scalar(box['box_pred_class_id']))
                    if k is not None:
                        ck.append(base + k)
                        cc.append(box['box_coords'])
                        cs.append(box['box_score'])
                elif t == 'gt':
                    k = cidx.get(_scalar(box['box_label']))
                    if k is not None:
                        gk.append(base + k)
                        gc.append(box['box_coords'])
            e += 1
    widths = {len(c) for c in cc} | {len(c) for c in gc}
    if not widths <= {4, 6} or len(widths) > 1:
        raise ValueError("box_coords must all have 4 (2D) or 6 (3D) entries, got lengths %s" % sorted(widths))
    dim = 2 if widths == {4} else 3
    n_groups = e * nc

    def grouped(keys, coords, scores=None):
        keys = np.asarray(keys, dtype=np.int64)
        order = np.argsort(keys, kind='stable')
        boxes = np.asarray(coords, dtype=np.float64).reshape(len(keys), 2 * dim)[order]
        off = np.zeros(n_groups + 1, dtype=np.int32)
        off[1:] = np.cumsum(np.bincount(keys, minlength=n_groups))
        sc = None if scores is None else np.asarray(scores, dtype=np.float64)[order]
        return boxes, sc, off

    cand, score, cand_off = grouped(ck, cc, cs)
    gt, _, gt_off = grouped(gk, gc)
    elem_off = np.zeros(len(n_elem) + 1, dtype=np.int32)
    elem_off[1:] = np.cumsum(n_elem)
    return dim, cand, score, cand_off, gt, gt_off, elem_off


def match_rows(flat, n_classes, ious):
    """mdt_eval_match on a flattened results list: (row_score fp64, row_meta int32 [n, 4] = type, class index, patient index, IoU index)"""
    dim, cand, score, cand_off, gt, gt_off, elem_off = flat
    n_pat, n_iou = elem_off.size - 1, len(ious)
    if n_pat == 0:
        return np.zeros(0), np.zeros((0, 4), dtype=np.int32)
    dev = _device()
    lib = L.load()
    n_cand, n_gt = cand.shape[0], gt.shape[0]
    max_rows = n_iou * (n_cand + n_gt + n_classes * n_pat)
    d = [_dev(x, dev, dt) for x, dt in ((cand, np.float64), (score, np.float64), (cand_off, np.int32), (gt, np.float64), (gt_off, np.int32),
                                        (elem_off, np.int32), (np.asarray(ious, dtype=np.float64), np.float64))]
    out = _Outputs(dev, [('n', np.int32, 1), ('score', np.float64, max_rows), ('meta', np.int32, 4 * max_rows)])
    ws = _workspace(lib.mdt_eval_match_workspace_bytes(n_iou * n_classes * n_pat, n_cand, n_gt, n_iou), dev)
    L.check(lib.mdt_eval_match(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), n_cand, L.ptr(d[3]), L.ptr(d[4]), n_gt, L.ptr(d[5]), n_pat, n_classes,
                               dim, L.ptr(d[6]), n_iou, out.ptr('score'), out.ptr('meta'), out.ptr('n'), L.ptr(ws), ws.numel(), L.stream_ptr()))
    h = out.fetch()
    n = int(h['n'][0])
    return h['score'][:n].copy(), h['meta'].reshape(-1, 4)[:n].copy()


def draw_multiplicities(n_pat, n_resamples, seed):
    """[n_resamples, n_pat] int32: row b is np.bincount of RandomState([seed, b]).randint(0, n_pat, n_pat), the patient multiplicities of
    bootstrap resample b (independent of n_resamples)"""
    mult = np.empty((n_resamples, n_pat), dtype=np.int32)
    for b in range(n_resamples):
        mult[b] = np.bincount(np.random.RandomState([seed, b]).randint(0, n_pat, size=n_pat), minlength=n_pat)
    return mult


def bootstrap_interval(values, alpha):
    """(lo, hi, n_valid): np.percentile(valid, [100 alpha / 2, 100 (1 - alpha / 2)]) over the non-NaN values (NaN, NaN when none)"""
    v = np.asarray(values, dtype=np.float64).reshape(-1)
    valid = v[~np.isnan(v)]
    if valid.size == 0:
        return np.nan, np.nan, 0
    lo, hi = np.percentile(valid, [100 * alpha / 2, 100 * (1 - alpha / 2)])
    return float(lo), float(hi), int(valid.size)


def _type_codes(det_type):
    codes = np.full(len(det_type), -1, dtype=np.int32)
    for k, t in enumerate(TYPES):
        codes[det_type == t] = k
    return codes


class Evaluator():

    def __init__(self, cf, logger, mode='test'):
        """mode: 'train', 'val_sampling', 'val_patient' or 'test' (the form of the results list, see evaluate_predictions)"""
        self.cf = cf
        self.logger = logger
        self.mode = mode
        self._cols = None
        self._df = None

    # ---------------------------------------------------------------------------------------------------------------- the rows
    @property
    def columns(self):
        """the columns of test_df as numpy arrays (pred_score, class_label, pred_class, pid, det_type, fold, match_iou); needs no pandas"""
        return self._cols

    @property
    def test_df(self):
        """the rows as the reference's pandas DataFrame (built on first access)"""
        if self._df is None and self._cols is not None:
            import pandas as pd
            c = self._cols
            df = pd.DataFrame()
            det = (c['det_type'] == 'det_tp') | (c['det_type'] == 'det_fp')
            # the reference's list mixes detection scores with integer zeros: an integer column when there is no detection row
            df['pred_score'] = c['pred_score'] if det.any() else c['pred_score'].astype(np.int64)
            df['class_label'] = c['class_label']
            df['pred_class'] = c['pred_class'].tolist()
            df['pid'] = c['pid'].tolist()
            df['det_type'] = c['det_type'].tolist()
            df['fold'] = self._fold_scalar
            df['match_iou'] = c['match_iou']
            self._df = df
        return self._df

    @test_df.setter
    def test_df(self, df):
        self._df = df
        self._cols = {'pred_score': df['pred_score'].to_numpy(np.float64), 'class_label': df['class_label'].to_numpy(np.int64),
                      'pred_class': df['pred_class'].to_numpy(), 'pid': df['pid'].to_numpy(object),
                      'det_type': df['det_type'].to_numpy(object), 'fold': df['fold'].to_numpy(object),
                      'match_iou': df['match_iou'].to_numpy(np.float64)}

    def evaluate_predictions(self, results_list, monitor_metrics=None):
        """Matches the predicted boxes to the ground-truth boxes for every match IoU in cf.ap_match_ious and every class of cf.class_dict,
        and stores one row per detection, missed GT box and empty patient (test_df / columns).
        results_list: in 'train' / 'val_sampling' mode [[[boxes_0, ...], [pid_0, ...]], ...] (batches of elements, scored one element at a
        time); otherwise [[elements_of_patient, pid], ...].  With monitor_metrics, returns return_metrics(monitor_metrics)."""
        self.logger.info('evaluating in mode {}'.format(self.mode))
        if self.mode == 'train' or self.mode == 'val_sampling':
            batch_elements_list = [[b_box_list] for item in results_list for b_box_list in item[0]]
            pid_list = [pid for item in results_list for pid in item[1]]
        else:
            batch_elements_list = [item[0] for item in results_list]
            pid_list = [item[1] for item in results_list]
        for match_iou in self.cf.ap_match_ious:
            self.logger.info('evaluating with match_iou: {}'.format(match_iou))
        classes = list(self.cf.class_dict.keys())
        ious = list(self.cf.ap_match_ious)
        score, meta = match_rows(flatten_results(batch_elements_list, classes), len(classes), ious)
        types = meta[:, 0]
        pids = np.empty(len(pid_list), dtype=object)
        pids[:] = pid_list
        self._fold_scalar = self.cf.fold
        fold = np.empty(types.size, dtype=object)
        fold[:] = [self.cf.fold] * types.size
        self._df = None
        self._cols = {'pred_score': score, 'class_label': ((types == 0) | (types == 2)).astype(np.int64),
                      'pred_class': np.asarray(classes)[meta[:, 1]], 'pid': pids[meta[:, 2]], 'det_type': _TYPES_ARR[types], 'fold': fold,
                      'match_iou': np.asarray(ious, dtype=np.float64)[meta[:, 3]]}
        if monitor_metrics is not None:
            return self.return_metrics(monitor_metrics)

    # ------------------------------------------------------------------------------------------------------------- the metrics
    def return_metrics(self, monitor_metrics=None):
        """AP / AUC per class and score level (cf.report_score_level) of the stored rows, plus the average foreground ROI AP.
        Returns (all_stats, monitor_metrics) as the reference does; with monitor_metrics, this epoch's values are appended to it.  Writes the
        prediction histograms and stat curves cf asks for into cf.plot_dir when that is a directory (see the module docstring)."""
        cf, c = self.cf, self._cols
        classes = list(cf.class_dict.keys())
        folds = _unique_in_order(c['fold'])[0]
        multi_fold = len(folds) > 1
        codes = _type_codes(c['det_type'])
        levels = list(cf.report_score_level)
        roi, pat = _RoiJobs(c, codes, cf.per_patient_ap), _PatientJobs(c)
        thresholds = [cf.min_det_thresh] + (SCAN_THRESHOLDS if cf.scan_det_thresh else [])
        for cl in classes:
            cmask = c['pred_class'] == cl
            if 'rois' in levels:
                spec = cmask & (codes != 3)
                roi.add(('all', cl), spec)
                if multi_fold:
                    for f in folds:
                        roi.add((f, cl), spec & (c['fold'] == f))
            if 'patient' in levels:
                pat.add_class(cl, cmask, folds if multi_fold else ())
        res = _run_metric_kernels(roi, pat, thresholds)
        plot_dir = getattr(cf, 'plot_dir', None)
        if plot_dir is not None and not os.path.isdir(plot_dir):
            plot_dir = None

        all_stats = []
        for cl in classes:
            for score_level in levels:
                stats_dict = {'name': 'fold_{} {} cl_{}'.format(cf.fold, score_level, cl)}
                if score_level == 'rois':
                    stats_dict['ap'] = roi.ap(res, ('all', cl), 0)
                    stats_dict['auc'] = 0
                    stats_dict['roc'] = None
                    stats_dict['prc'] = None
                    if multi_fold:
                        stats_dict['mean_ap'] = np.mean([roi.ap(res, (f, cl), 0) for f in folds])
                        stats_dict['mean_auc'] = 0
                if score_level == 'patient':
                    auc, roc, ap, prc = pat.scores(res, ('all', cl))
                    stats_dict['auc'], stats_dict['roc'], stats_dict['ap'], stats_dict['prc'] = auc, roc, ap, prc
                    if multi_fold:
                        aucs, aps = [], []
                        for f in folds:
                            fa, _, fp, _ = pat.scores(res, (f, cl))
                            if not (isinstance(fa, float) and np.isnan(fa)):
                                aucs.append(fa)
                            if not (isinstance(fp, float) and np.isnan(fp)):
                                aps.append(fp)
                        stats_dict['mean_auc'] = np.mean(aucs)
                        stats_dict['mean_ap'] = np.mean(aps)
                if monitor_metrics is not None and not (score_level == 'patient' and cl != cf.patient_class_of_interest):
                    score_level_name = 'patient' if score_level == 'patient' else cf.class_dict[cl]
                    monitor_metrics[score_level_name + '_ap'].append(stats_dict['ap'] if stats_dict['ap'] > 0 else None)
                    if score_level == 'patient':
                        monitor_metrics[score_level_name + '_auc'].append(stats_dict['auc'] if stats_dict['auc'] > 0 else None)
                if plot_dir is not None and cf.plot_prediction_histograms:
                    self._plot_hist(plot_dir, cl, score_level, codes)
                all_stats.append(stats_dict)
                if cf.scan_det_thresh and score_level == 'rois':
                    aps = [roi.ap(res, ('all', cl), 1 + k) for k in range(len(SCAN_THRESHOLDS))]
                    self.logger.info('results from scanning over det_threshs: {}'.format([[i, j] for i, j in zip(SCAN_THRESHOLDS, aps)]))

        if plot_dir is not None and cf.plot_stat_curves:
            plotting.plot_stat_curves(all_stats, os.path.join(plot_dir, '{}_{}_stat_curves'.format(cf.fold, self.mode)))
        avg_ap = np.mean([d['ap'] for d in all_stats if 'rois' in d['name']])
        all_stats.append({'name': 'average_foreground_roi', 'auc': 0, 'ap': avg_ap})
        if multi_fold:
            all_stats[-1]['mean_ap'] = np.mean([d['mean_ap'] for d in all_stats if 'rois' in d['name']])
            all_stats[-1]['mean_auc'] = 0
        # identical model-selection values across epochs break the checkpoint ranking: perturb a repeated value (numpy's global RNG)
        for sc in cf.model_selection_criteria:
            if 'val' in self.mode and monitor_metrics[sc].count(monitor_metrics[sc][-1]) > 1 and monitor_metrics[sc][-1] is not None:
                monitor_metrics[sc][-1] += 1e-6 * np.random.rand()
        return all_stats, monitor_metrics

    def _plot_hist(self, plot_dir, cl, score_level, codes):
        """the reference's prediction histogram of one class and score level: the ROI rows without patient_tn dummies (with their types), or
        per patient (sorted pids) the max label and max score"""
        c = self._cols
        cmask = c['pred_class'] == cl
        if score_level == 'rois':
            spec = cmask & (codes != 3)
            labels, preds, types = c['class_label'][spec].tolist(), c['pred_score'][spec].tolist(), c['det_type'][spec].tolist()
        else:
            idx = np.nonzero(cmask)[0]
            _, inv = np.unique(c['pid'][idx], return_inverse=True)
            inv = inv.reshape(-1)
            n = int(inv.max()) + 1 if idx.size else 0
            lab, sc = np.full(n, np.iinfo(np.int64).min, np.int64), np.full(n, -np.inf)
            np.maximum.at(lab, inv, c['class_label'][idx])
            np.maximum.at(sc, inv, c['pred_score'][idx])
            labels, preds, types = lab.tolist(), sc.tolist(), None
        name = 'pred_hist_{}_{}_{}_cl{}'.format(self.cf.fold, 'val' if 'val' in self.mode else self.mode, score_level, cl)
        plotting.plot_prediction_hist(labels, preds, types, os.path.join(plot_dir, name))

    def score_test_df(self, internal_df=True):
        """Writes this fold's rows to <exp_dir>/<fold>_test_df.pickle and its scores to results.txt; once cf.n_cv_splits fold pickles exist,
        also scores the folds' aggregate into results.txt and ../results_table.txt (the reference's files and text)."""
        import pandas as pd
        cf = self.cf
        if internal_df:
            self.test_df.to_pickle(os.path.join(cf.exp_dir, '{}_test_df.pickle'.format(cf.fold)))
            stats, _ = self.return_metrics()
            with open(os.path.join(cf.exp_dir, 'results.txt'), 'a') as handle:
                handle.write('\n****************************\n')
                handle.write('\nresults for fold {} \n'.format(cf.fold))
                handle.write('\n****************************\n')
                handle.write('\nfold df shape {}\n  \n'.format(self.test_df.shape))
                for s in stats:
                    handle.write('AUC {:0.4f}  AP {:0.4f} {} \n'.format(s['auc'], s['ap'], s['name']))
        fold_df_paths = [ii for ii in os.listdir(cf.exp_dir) if 'test_df.pickle' in ii]
        if len(fold_df_paths) == cf.n_cv_splits:
            with open(os.path.join(cf.exp_dir, 'results.txt'), 'a') as handle:
                cf.fold = 'overall'
                dfs_list = [pd.read_pickle(os.path.join(cf.exp_dir, ii)) for ii in fold_df_paths]
                for ix, df in enumerate(dfs_list):
                    df['fold'] = ix
                self.test_df = pd.concat(dfs_list)
                stats, _ = self.return_metrics()
                handle.write('\n****************************\n')
                handle.write('\nOVERALL RESULTS \n')
                handle.write('\n****************************\n')
                handle.write('\ndf shape \n  \n')        # the reference's format string has no placeholder for the shape
                for s in stats:
                    handle.write('\nAUC {:0.4f} (mu {:0.4f})  AP {:0.4f} (mu {:0.4f})  {}\n '
                                 .format(s['auc'], s['mean_auc'], s['ap'], s['mean_ap'], s['name']))
                results_table_path = os.path.join(("/").join(cf.exp_dir.split("/")[:-1]), 'results_table.txt')
                with open(results_table_path, 'a') as handle2:
                    for s in stats:
                        handle2.write('\nAUC {:0.4f} (mu {:0.4f})  AP {:0.4f} (mu {:0.4f})  {} {}'
                                      .format(s['auc'], s['mean_auc'], s['ap'], s['mean_ap'], s['name'], cf.exp_dir.split('/')[-1]))
                    handle2.write('\n')

    # ------------------------------------------------------------------------------------------------------- bootstrap and FROC
    def bootstrap(self, n_resamples=1000, seed=0, alpha=0.05, fps_per_scan=FROC_RATES):
        """Patient-bootstrap confidence intervals of the stored rows' metrics, with FROC and CPM.

        The units are the distinct pids of the rows (np.unique order; several folds' rows are pooled), P of them.  Resample b draws
        RandomState([seed, b]).randint(0, P, P), so it does not depend on n_resamples; patient p then weighs m[p] = its draw count.  A
        resample's metrics are those of the materialised resample: every row of p repeated m[p] times in place, copy j of p a patient of
        its own, the matching not redone.  The kernels (mdt_eval_bootstrap_roi / _patient) compute them from integer weighted counts,
        bit-identical to the materialised evaluation, and the host applies return_metrics' expressions to their outputs:
          - ROI AP per class: the mean over the match-IoU segments with all_p > 0 of the 101-point interpolated precision at
            cf.min_det_thresh (cf.per_patient_ap is not used); average_foreground_roi is the mean over the classes of each resample;
          - patient AUC / AP per class: return_metrics' curve expressions on the weighted distinct-threshold counts;
          - FROC per class and match IoU: sens(r) = max{TP(v) : FP(v) <= r * P} / G over the operating points (the origin and, per
            distinct score v above cf.min_det_thresh, the TP / FP detections with score >= v; NaN scores left out), G the det_tp + det_fn
            rows, NaN when G = 0.  This is the step FROC: LUNA16's script interpolates linearly between operating points, this one
            does not.  The CPM is the mean of sens over fps_per_scan.
        The interval of each metric is np.percentile(valid, [100 alpha / 2, 100 (1 - alpha / 2)]) over the resamples where it is not
        NaN, n_valid their number.  The point estimate is the metric of the rows themselves (every m = 1).

        Returns a list of dicts named like return_metrics' entries ('fold_{} rois cl_{}', 'fold_{} patient cl_{}',
        'average_foreground_roi'): 'ap' (and 'auc' at the patient level) and, per match IoU of a 'rois' entry, 'froc'[iou] = {'sens':
        one stat per rate, 'cpm': stat}, each stat {'value': point estimate, 'ci': (lo, hi), 'n_valid': n}.  The per-resample values are
        kept in self.bootstrap_values (same names, numpy arrays).  n_resamples = 0 gives the point estimates alone."""
        c, cf = self._cols, self.cf
        if c is None or c['pred_score'].size == 0:
            raise ValueError("bootstrap: no rows are stored (run evaluate_predictions or set test_df first)")
        if isinstance(n_resamples, bool) or not isinstance(n_resamples, (int, np.integer)) or n_resamples < 0:
            raise ValueError("bootstrap: n_resamples must be an integer >= 0, got %r" % (n_resamples,))
        if not 0 < alpha < 1:
            raise ValueError("bootstrap: alpha must lie in (0, 1), got %r" % (alpha,))
        rates = np.asarray(fps_per_scan, dtype=np.float64).reshape(-1)
        if rates.size == 0 or not np.all(np.isfinite(rates) & (rates > 0)):
            raise ValueError("bootstrap: fps_per_scan must be positive finite rates, got %r" % (fps_per_scan,))
        n_resamples = int(n_resamples)
        classes = list(cf.class_dict.keys())
        levels = list(cf.report_score_level)
        roi, pat, pat_idx, n_pat = _bootstrap_jobs(c, classes, levels)
        mult = np.concatenate([np.ones((1, n_pat), dtype=np.int32), draw_multiplicities(n_pat, n_resamples, seed)])
        roi_ious = {key: _unique_in_order(c['match_iou'][idx])[0] for key, idx in zip(roi.jobs, roi.rows)}
        n_members = sum(m.size for m in pat.members)
        per_resample = roi.n_seg * (8 * RECALL_POINTS.size + 4 * (2 + rates.size)) + 16 * n_members + 4 * len(pat.members)
        chunk = max(1, BOOTSTRAP_CHUNK_BYTES // max(per_resample, 1))

        names = []
        vals = {}
        for cl in classes:
            for level in levels:
                name = 'fold_{} {} cl_{}'.format(cf.fold, level, cl)
                names.append((name, level, cl))
                if level == 'rois':
                    vals[name] = {'ap': [], 'froc': {float(i): {'sens': [], 'cpm': []} for i in roi_ious[('all', cl)]}}
                else:
                    vals[name] = {'auc': [], 'ap': []}
        vals['average_foreground_roi'] = {'ap': []}
        for s0 in range(0, 1 + n_resamples, chunk):
            res = _run_bootstrap_kernels(roi, pat, pat_idx, n_pat, mult[s0:s0 + chunk], cf.min_det_thresh, rates * n_pat)
            for b in range(min(chunk, 1 + n_resamples - s0)):
                roi_aps = []
                for name, level, cl in names:
                    v = vals[name]
                    if level == 'rois':
                        q, counts = res['q'][b][:, None, :], res['counts'][b]
                        ap = roi.ap({'q': q, 'counts': counts}, ('all', cl), 0)
                        v['ap'].append(ap)
                        roi_aps.append(ap)
                        base, n = roi.jobs[('all', cl)]
                        for s, iou in zip(range(base, base + n), v['froc']):
                            g = counts[s, 0]
                            sens = res['froc'][b][s] / np.float64(g) if g > 0 else np.full(rates.size, np.nan)
                            v['froc'][iou]['sens'].append(sens)
                            v['froc'][iou]['cpm'].append(np.mean(sens))
                    else:
                        auc, _, ap, _ = pat.scores({k: res[k][b] for k in ('thr', 'tps', 'fps', 'n_thr')}, ('all', cl))
                        v['auc'].append(auc)
                        v['ap'].append(ap)
                vals['average_foreground_roi']['ap'].append(np.mean(roi_aps))

        def stat(x):
            x = np.asarray(x, dtype=np.float64)
            lo, hi, n_valid = bootstrap_interval(x[1:], alpha)
            return {'value': x[0], 'ci': (lo, hi), 'n_valid': n_valid}

        stats, self.bootstrap_values = [], {}
        for name, v in list(vals.items()):
            entry, raw = {'name': name}, {}
            for k in ('auc', 'ap'):
                if k in v:
                    entry[k], raw[k] = stat(v[k]), np.asarray(v[k], dtype=np.float64)[1:]
            if 'froc' in v:
                entry['fps_per_scan'] = tuple(rates.tolist())
                entry['froc'], raw['froc'] = {}, {}
                for iou, f in v['froc'].items():
                    sens = np.asarray(f['sens'], dtype=np.float64).reshape(-1, rates.size)
                    entry['froc'][iou] = {'sens': [stat(sens[:, k]) for k in range(rates.size)], 'cpm': stat(f['cpm'])}
                    raw['froc'][iou] = {'sens': sens[1:], 'cpm': np.asarray(f['cpm'], dtype=np.float64)[1:]}
            stats.append(entry)
            self.bootstrap_values[name] = raw
        return stats

    def score_bootstrap(self, n_resamples=1000, seed=0, alpha=0.05, fps_per_scan=FROC_RATES):
        """bootstrap() of the stored rows, appended as text to <exp_dir>/results_bootstrap.txt, one line per metric:
        '<metric> <point> [<lo>, <hi>] (n <n_valid>) <name>[ iou <match iou>]'.  Returns the stats."""
        stats = self.bootstrap(n_resamples, seed, alpha, fps_per_scan)
        n_pat = np.unique(self._cols['pid']).size

        def line(metric, s, name):
            return '{} {:0.4f} [{:0.4f}, {:0.4f}] (n {}) {}\n'.format(metric, s['value'], s['ci'][0], s['ci'][1], s['n_valid'], name)
        with open(os.path.join(self.cf.exp_dir, 'results_bootstrap.txt'), 'a') as handle:
            handle.write('\n****************************\n')
            handle.write('\nbootstrap of fold {}: {} patients, {} resamples, seed {}, {:g}% intervals\n\n'
                         .format(self.cf.fold, n_pat, n_resamples, seed, 100 * (1 - alpha)))
            for s in stats:
                for k in ('auc', 'ap'):
                    if k in s:
                        handle.write(line(k.upper(), s[k], s['name']))
                for iou, f in s.get('froc', {}).items():
                    for r, st in zip(s['fps_per_scan'], f['sens']):
                        handle.write(line('FROC@{:g}'.format(r), st, '{} iou {:g}'.format(s['name'], iou)))
                    handle.write(line('CPM', f['cpm'], '{} iou {:g}'.format(s['name'], iou)))
        return stats


# ---------------------------------------------------------------------------------------------------------------- metric plumbing
class _RoiJobs:
    """ROI-AP segments: per job (a class, all rows or one fold) the segments (IoU) or (IoU, pid) in get_roi_ap_from_df's loop order"""

    def __init__(self, cols, codes, per_patient):
        self.c, self.codes, self.per_patient = cols, codes, bool(per_patient)
        self.jobs, self.rows, self.segs, self.n_seg = {}, [], [], 0

    def add(self, key, mask):
        idx = np.nonzero(mask)[0]
        _, iou_inv = _unique_in_order(self.c['match_iou'][idx])
        n_iou = int(iou_inv.max()) + 1 if idx.size else 0
        if self.per_patient and idx.size:
            _, pid_inv = _unique_in_order(self.c['pid'][idx])
            n_pid = int(pid_inv.max()) + 1
            seg, n = iou_inv * n_pid + pid_inv, n_iou * n_pid
        else:
            seg, n = iou_inv, n_iou
        self.jobs[key] = (self.n_seg, n)
        self.rows.append(idx)
        self.segs.append(seg + self.n_seg)
        self.n_seg += n

    def ap(self, res, key, ti):
        """get_roi_ap_from_df at threshold index ti: np.mean over the segments' APs, each the np.mean of 101 interpolated precisions"""
        base, n = self.jobs[key]
        q, counts = res['q'], res['counts']
        aps = []
        for s in range(base, base + n):
            all_p, nd = counts[s, 0], counts[s, 1 + ti]
            if self.per_patient:
                if nd == 0 and all_p == 0:
                    continue
                aps.append(0 if all_p == 0 else np.mean(q[s, ti]))
            elif all_p > 0:
                aps.append(np.mean(q[s, ti]))
        return np.mean(aps)


class _PatientJobs:
    """patient-level segments: the (class, pid) slots of a class (groupby('pid'): sorted pids), all of them or those of one fold"""

    def __init__(self, cols):
        self.c = cols
        self.row_slot = np.full(cols['pred_score'].size, -1, dtype=np.int32)
        self.n_slots, self.jobs, self.members = 0, {}, []

    def add_class(self, cl, cmask, folds):
        idx = np.nonzero(cmask)[0]
        _, first, inv = np.unique(self.c['pid'][idx], return_index=True, return_inverse=True)
        slots = self.n_slots + np.arange(first.size, dtype=np.int32)
        self.row_slot[idx] = self.n_slots + inv.reshape(-1)
        self.n_slots += first.size
        self._add(('all', cl), slots)
        slot_fold = self.c['fold'][idx[first]]                      # agg({'fold': 'first'})
        for f in folds:
            self._add((f, cl), slots[slot_fold == f])

    def _add(self, key, slots):
        off = sum(m.size for m in self.members)
        self.jobs[key] = (len(self.members), off)
        self.members.append(slots)

    def scores(self, res, key):
        """(auc, roc, ap, prc) of one segment from its distinct-threshold counts: scikit-learn 1.9's roc_auc_score, roc_curve,
        average_precision_score and precision_recall_curve expressions; NaN where the reference's guards give NaN"""
        k, off = self.jobs[key]
        n = int(res['n_thr'][k])
        thr = res['thr'][off:off + n]
        tps = res['tps'][off:off + n].astype(np.float64)
        fps = res['fps'][off:off + n].astype(np.float64)
        auc = roc = ap = prc = np.nan
        if n and tps[-1] > 0 and fps[-1] > 0:
            f, t, th = fps, tps, thr
            if f.shape[0] > 2:                                            # drop_intermediate
                keep = np.where(np.concatenate([[True], np.logical_or(np.diff(f, 2), np.diff(t, 2)), [True]]))[0]
                f, t, th = f[keep], t[keep], th[keep]
            t = np.concatenate([[0.0], t])
            f = np.concatenate([[0.0], f])
            th = np.concatenate([[np.inf], th.astype(np.float64)])
            fpr, tpr = f / f[-1], t / t[-1]
            roc = (fpr, tpr, th)
            d = fpr[1:] - fpr[:-1]                                        # fpr ascends: auc's direction is 1
            auc = float(np.sum(d * (tpr[1:] + tpr[:-1]) / 2.0, dtype=np.float64))
        if n and tps[-1] > 0:
            ps = tps + fps
            precision = np.where(ps != 0, np.divide(tps, ps), 0.0)
            recall = tps / tps[-1]
            prc = (np.concatenate((np.flip(precision), [1.0])), np.concatenate((np.flip(recall), [0.0])), np.flip(thr))
            ap = float(max(0.0, -np.sum(np.diff(prc[1]) * prc[0][:-1])))
        return auc, roc, ap, prc


def _run_metric_kernels(roi, pat, thresholds):
    """mdt_eval_roi_ap and mdt_eval_patient on the stored rows; their outputs share one device buffer and return in one copy"""
    c = roi.c
    dev = _device()
    lib = L.load()
    stream = L.stream_ptr()
    n_thr = len(thresholds)
    n_members = sum(m.size for m in pat.members)
    specs = []
    if roi.n_seg:
        specs += [('q', np.float64, roi.n_seg * n_thr * RECALL_POINTS.size), ('counts', np.int32, roi.n_seg * (1 + n_thr))]
    if pat.members:
        specs += [('thr', np.float64, n_members), ('tps', np.int32, n_members), ('fps', np.int32, n_members), ('n_thr', np.int32, len(pat.members))]
    if not specs:
        return {}
    out = _Outputs(dev, specs)
    keep = []
    if roi.n_seg:
        idx = np.concatenate(roi.rows)
        n = int(idx.size)
        score = _dev(c['pred_score'][idx], dev, np.float64)
        seg = _dev(np.concatenate(roi.segs), dev, np.int32)
        kind = _dev(roi.codes[idx], dev, np.int32)
        th = _dev(np.asarray(thresholds, dtype=np.float64), dev, np.float64)
        rp = _dev(RECALL_POINTS, dev, np.float64)
        ws = _workspace(lib.mdt_eval_roi_ap_workspace_bytes(max(n, 1), roi.n_seg), dev)
        keep += [score, seg, kind, th, rp, ws]
        L.check(lib.mdt_eval_roi_ap(L.ptr(score), L.ptr(seg), L.ptr(kind), n, roi.n_seg, L.ptr(th), n_thr, L.ptr(rp), RECALL_POINTS.size,
                                    out.ptr('q'), out.ptr('counts'), L.ptr(ws), ws.numel(), stream))
    if pat.members:
        n = int(c['pred_score'].size)
        score = _dev(c['pred_score'], dev, np.float64)
        label = _dev(c['class_label'], dev, np.int32)
        slot = _dev(pat.row_slot, dev, np.int32)
        seg_off = np.zeros(len(pat.members) + 1, dtype=np.int32)
        seg_off[1:] = np.cumsum([m.size for m in pat.members])
        so = _dev(seg_off, dev, np.int32)
        ss = _dev(np.concatenate(pat.members) if n_members else np.zeros(1), dev, np.int32)
        ws = _workspace(lib.mdt_eval_patient_workspace_bytes(max(pat.n_slots, 1), n_members), dev)
        keep += [score, label, slot, so, ss, ws]
        L.check(lib.mdt_eval_patient(L.ptr(score), L.ptr(label), L.ptr(slot), n, max(pat.n_slots, 1), L.ptr(so), L.ptr(ss), n_members,
                                     len(pat.members), out.ptr('thr'), out.ptr('tps'), out.ptr('fps'), out.ptr('n_thr'), L.ptr(ws), ws.numel(),
                                     stream))
    res = out.fetch()
    if 'counts' in res:
        res['q'] = res['q'].reshape(roi.n_seg, n_thr, RECALL_POINTS.size)
        res['counts'] = res['counts'].reshape(roi.n_seg, 1 + n_thr)
    return res


def _bootstrap_jobs(c, classes, levels):
    """(roi, pat, patient index per row, P): one ROI job per class (segments = match IoUs) and one patient job per class, folds pooled"""
    _, pat_idx = np.unique(c['pid'], return_inverse=True)
    pat_idx = pat_idx.reshape(-1)
    codes = _type_codes(c['det_type'])
    roi, pat = _RoiJobs(c, codes, False), _PatientJobs(c)
    for cl in classes:
        cmask = c['pred_class'] == cl
        if 'rois' in levels:
            roi.add(('all', cl), cmask & (codes != 3))
        if 'patient' in levels:
            pat.add_class(cl, cmask, ())
    return roi, pat, pat_idx, int(pat_idx.max()) + 1


def _run_bootstrap_kernels(roi, pat, pat_idx, n_pat, mult, threshold, fp_limits):
    """mdt_eval_bootstrap_roi and mdt_eval_bootstrap_patient for the resamples mult [n_boot, n_pat]; one device buffer, one copy back"""
    c = roi.c
    dev = _device()
    lib = L.load()
    stream = L.stream_ptr()
    n_boot, n_r, n_rates = mult.shape[0], RECALL_POINTS.size, fp_limits.size
    n_members = sum(m.size for m in pat.members)
    specs = []
    if roi.n_seg:
        specs += [('q', np.float64, n_boot * roi.n_seg * n_r), ('counts', np.int32, n_boot * roi.n_seg * 2),
                  ('froc', np.int32, n_boot * roi.n_seg * n_rates)]
    if pat.members:
        specs += [('thr', np.float64, n_boot * n_members), ('tps', np.int32, n_boot * n_members), ('fps', np.int32, n_boot * n_members),
                  ('n_thr', np.int32, n_boot * len(pat.members))]
    if not specs:
        return {}
    out = _Outputs(dev, specs)
    m = _dev(mult, dev, np.int32)
    keep = [m]
    if roi.n_seg:
        idx = np.concatenate(roi.rows)
        n = int(idx.size)
        d = [_dev(c['pred_score'][idx], dev, np.float64), _dev(np.concatenate(roi.segs), dev, np.int32), _dev(roi.codes[idx], dev, np.int32),
             _dev(pat_idx[idx], dev, np.int32), _dev(RECALL_POINTS, dev, np.float64), _dev(fp_limits, dev, np.float64)]
        ws = _workspace(lib.mdt_eval_bootstrap_roi_workspace_bytes(max(n, 1), roi.n_seg, n_pat), dev)
        keep += d + [ws]
        L.check(lib.mdt_eval_bootstrap_roi(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), n, roi.n_seg, n_pat, L.ptr(m), n_boot,
                                           float(threshold), L.ptr(d[4]), n_r, L.ptr(d[5]), n_rates, out.ptr('q'), out.ptr('counts'),
                                           out.ptr('froc'), L.ptr(ws), ws.numel(), stream))
    if pat.members:
        n = int(c['pred_score'].size)
        seg_off = np.zeros(len(pat.members) + 1, dtype=np.int32)
        seg_off[1:] = np.cumsum([s.size for s in pat.members])
        d = [_dev(c['pred_score'], dev, np.float64), _dev(c['class_label'], dev, np.int32), _dev(pat.row_slot, dev, np.int32),
             _dev(pat_idx, dev, np.int32), _dev(seg_off, dev, np.int32),
             _dev(np.concatenate(pat.members) if n_members else np.zeros(1), dev, np.int32)]
        ws = _workspace(lib.mdt_eval_bootstrap_patient_workspace_bytes(max(pat.n_slots, 1), n_members, len(pat.members)), dev)
        keep += d + [ws]
        L.check(lib.mdt_eval_bootstrap_patient(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), n, max(pat.n_slots, 1), L.ptr(d[4]),
                                               L.ptr(d[5]), n_members, len(pat.members), n_pat, L.ptr(m), n_boot, out.ptr('thr'),
                                               out.ptr('tps'), out.ptr('fps'), out.ptr('n_thr'), L.ptr(ws), ws.numel(), stream))
    res = out.fetch()
    if roi.n_seg:
        res['q'] = res['q'].reshape(n_boot, roi.n_seg, n_r)
        res['counts'] = res['counts'].reshape(n_boot, roi.n_seg, 2)
        res['froc'] = res['froc'].reshape(n_boot, roi.n_seg, n_rates)
    if pat.members:
        for k in ('thr', 'tps', 'fps'):
            res[k] = res[k][:n_boot * n_members].reshape(n_boot, n_members) if n_members else np.zeros((n_boot, 0), res[k].dtype)
        res['n_thr'] = res['n_thr'].reshape(n_boot, len(pat.members))
    return res
