"""Generates tests/golden/plot_calls.pkl.gz: the matplotlib calls the reference's plotting.py makes on seeded inputs.

    python tests/golden/make_plot_golden.py <root of the reference medicaldetectiontoolkit checkout>

The reference's unmodified plotting.py is imported under a recording stand-in for matplotlib (pyplot, gridspec and the figure / axes
objects).  Every imshow, plot, hist, text, title, axis labels, limits, yscale, legend and savefig call is recorded with its arguments, in
order; each savefig stores the figure's calls so far.  The file holds, per case, the inputs and the saved figures (or the exception the
reference raised), so tests/test_plotting_cpu.py can run medicaldetectiontoolkit_b200.plotting on the same inputs and compare its content.
"""
import copy
import gzip
import importlib.util
import os
import pickle
import sys
import types

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'plot_calls.pkl.gz')


# ------------------------------------------------------------------------------------------------------------------ recording stub
class _Fig:
    def __init__(self, figsize):
        self.figsize = tuple(figsize) if figsize is not None else (6.4, 4.8)
        self.calls, self.gridspec = [], None

    def savefig(self, name):
        _REC.saved.append({'file': name, 'figsize': self.figsize, 'gridspec': self.gridspec, 'calls': copy.deepcopy(self.calls)})


class _Box:
    x0, y0, width, height = 0.125, 0.11, 0.9 - 0.125, 0.88 - 0.11


class _Ax:
    def __init__(self, fig):
        self.fig = fig

    def _r(self, *c):
        self.fig.calls.append(c)

    def axis(self, v):
        self._r('axis', v)

    def set_xlabel(self, s):
        self._r('xlabel', s)

    def set_ylabel(self, s):
        self._r('ylabel', s)

    def set_xlim(self, a, b):
        self._r('xlim', a, b)

    def set_ylim(self, a, b):
        self._r('ylim', a, b)

    def grid(self):
        self._r('grid')

    def plot(self, x, y, **kw):
        self._r('plot', copy.deepcopy(x), copy.deepcopy(y), kw)

    def get_position(self):
        return _Box()

    def set_position(self, pos):
        self._r('set_position', list(pos))

    def legend(self, **kw):
        self._r('legend', kw)

    def set_title(self, s, **kw):
        self._r('title', s, kw)


class _Rec:
    def __init__(self):
        self.saved, self.fig = [], None


_REC = _Rec()


class _GridSpec:
    def __init__(self, nrows, ncols):
        self.shape = (nrows, ncols)
        _REC.fig.gridspec = [nrows, ncols, {}]

    def update(self, **kw):
        _REC.fig.gridspec[2].update(kw)

    def __getitem__(self, k):
        return ('cell', k)


def _cur(*c):
    _REC.fig.calls.append(c)


def _figure(figsize=None):
    _REC.fig = _Fig(figsize)
    return _REC.fig


def _subplot(arg):
    _cur('subplot', arg[1] if isinstance(arg, tuple) else arg)
    return _Ax(_REC.fig)


def _make_stub():
    mpl = types.ModuleType('matplotlib')
    mpl.use = lambda *a, **k: None
    plt = types.ModuleType('matplotlib.pyplot')
    plt.figure = _figure
    plt.subplot = _subplot
    plt.title = lambda s, **kw: _cur('title', s, kw)
    plt.imshow = lambda arr, **kw: _cur('imshow', np.array(arr), kw)
    plt.plot = lambda x, y, **kw: _cur('plot', copy.deepcopy(x), copy.deepcopy(y), kw)
    plt.text = lambda x, y, s, **kw: _cur('text', x, y, s, kw)
    plt.hist = lambda d, **kw: _cur('hist', np.array(d), kw)
    plt.yscale = lambda v: _cur('yscale', v)
    plt.legend = lambda **kw: _cur('legend', kw)
    plt.xlabel = lambda s: _cur('xlabel', s)
    plt.ylabel = lambda s: _cur('ylabel', s)
    plt.savefig = lambda name: _REC.fig.savefig(name)
    plt.close = lambda *a: None
    gs = types.ModuleType('matplotlib.gridspec')
    gs.GridSpec = _GridSpec
    mpl.pyplot, mpl.gridspec = plt, gs
    sys.modules.update({'matplotlib': mpl, 'matplotlib.pyplot': plt, 'matplotlib.gridspec': gs})


# --------------------------------------------------------------------------------------------------------------------------- cases
class CF:
    def __init__(self, **kw):
        self.__dict__.update(kw)


PALETTE = {'det': 'b', 'gt': 'r', 'neg_class': 'purple', 'prop': 'w', 'pos_class': 'g', 'pos_anchor': 'c', 'neg_anchor': 'c'}


def _boxes(rs, dim, n_z, Y, X):
    def coords(z=True):
        y1, x1 = rs.randint(0, Y - 6), rs.randint(0, X - 6)
        c = [y1, x1, y1 + rs.randint(3, 6), x1 + rs.randint(3, 6)]
        if dim == 3 and z:
            z1 = rs.uniform(-1.5, n_z - 2)
            c += [z1, z1 + rs.uniform(0, 4)]
        return np.array(c, dtype=np.float64 if dim == 3 else np.int64)
    out = [{'box_coords': coords(), 'box_type': 'gt', 'box_label': 1},
           {'box_coords': coords(), 'box_type': 'gt', 'box_label': 2},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.87, 'box_pred_class_id': 1},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.454, 'box_pred_class_id': 2},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.05, 'box_pred_class_id': 1},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.9, 'box_pred_class_id': 0},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.6, 'box_pred_class_id': 1, 'sample_id': 0},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.7, 'box_pred_class_id': 2, 'sample_id': 1},
           {'box_coords': coords(), 'box_type': 'det', 'box_score': 0.33, 'box_pred_class_id': 1, 'extra_usage': 'pos_class'},
           {'box_coords': coords(), 'box_type': 'pos_anchor'}, {'box_coords': coords(), 'box_type': 'neg_anchor'},
           {'box_coords': coords(), 'box_type': 'prop'}, {'box_coords': coords(), 'box_type': 'patient_tn_box'}]
    return out


def batch_case(dim, B, C, Y, X, Z, n_cls, seed, same_pid=False, no_gt_in=()):
    rs = np.random.RandomState(seed)
    shp = (B, C, Y, X) + ((Z,) if dim == 3 else ())
    data = rs.randn(*shp).astype(np.float32)
    seg = rs.randint(0, n_cls, size=(B, 1) + shp[2:]).astype(np.uint8)
    seg_preds = rs.randint(0, n_cls, size=(B, 1) + shp[2:]).astype(np.int64)
    boxes = []
    for b in range(B):
        bl = _boxes(rs, dim, Z, Y, X)
        if b in no_gt_in:
            bl = [x for x in bl if x['box_type'] != 'gt']
        boxes.append(bl)
    pids = ['pid_%d_with_a_long_name' % (b if not same_pid else 7) for b in range(B)]
    cf = CF(dim=dim, num_seg_classes=n_cls, fold=2, plot_dir='/plots', box_color_palette=PALETTE)
    return {'batch': {'data': data, 'seg': seg, 'pid': pids}, 'results_dict': {'boxes': boxes, 'seg_preds': seg_preds}, 'cf': cf.__dict__,
            'seed': seed}


def run_batch(plotting, case):
    np.random.seed(case['seed'])
    plotting.plot_batch_prediction(copy.deepcopy(case['batch']), copy.deepcopy(case['results_dict']), CF(**case['cf']))


def hist_cases():
    rs = np.random.RandomState(5)
    n = 300
    labels = (rs.rand(n) < 0.3).astype(int).tolist()
    preds = rs.rand(n).tolist()
    types_ = [('det_tp' if l else 'det_fp') if rs.rand() < 0.8 else ('det_fn' if l else 'det_fp') for l in labels]
    return [dict(label_list=labels, pred_list=preds, type_list=types_, outfile='/plots/pred_hist_0_val_rois_cl1'),
            dict(label_list=labels, pred_list=preds, type_list=None, outfile='/plots/pred_hist_0_val_patient_cl1'),
            dict(label_list=[0] * 20, pred_list=rs.rand(20).tolist(), type_list=['det_fp'] * 20, outfile='/plots/only_fp'),
            dict(label_list=[1] * 5, pred_list=[0.0, 0.2, 0.2, 1.0, 0.5], type_list=['det_fn', 'det_tp', 'det_tp', 'det_tp', 'det_tp'],
                 outfile='/plots/only_tp')]


def stat_cases():
    fpr = np.array([0, 0, 0.25, 0.5, 1.0])
    tpr = np.array([0, 0.5, 0.5, 1.0, 1.0])
    thr = np.array([np.inf, 0.9, 0.6, 0.3, 0.1])
    prc = (np.array([0.5, 0.66, 1.0, 1.0]), np.array([1.0, 1.0, 0.5, 0.0]), np.array([0.1, 0.3, 0.9]))
    ok = [{'name': 'fold_0 patient cl_1', 'auc': 0.8, 'ap': 0.9, 'roc': (fpr, tpr, thr), 'prc': prc},
          {'name': 'fold_0 rois cl_1', 'auc': 0, 'ap': 0.5, 'roc': None, 'prc': None},
          {'name': 'fold_0 patient cl_2', 'auc': 0.6, 'ap': 0.7, 'roc': (tpr * 0.5, tpr, thr), 'prc': (prc[0][::-1], prc[1], prc[2])}]
    nan = ok + [{'name': 'fold_0 patient cl_3', 'auc': np.nan, 'ap': np.nan, 'roc': np.nan, 'prc': np.nan}]
    return [dict(stats=ok, outfile='/plots/0_val_sampling_stat_curves'), dict(stats=nan, outfile='/plots/0_test_stat_curves')]


def monitor_cases():
    rs = np.random.RandomState(9)
    out = []
    for do_val, n_fig, extra in ((True, 2, {1: ['class_loss']}), (False, 1, {})):
        cf = CF(plot_dir='/plots', fold=1, fold_dir='/exp/fold_1', do_validation=do_val, assign_values_to_extra_figure=extra,
                n_monitoring_figures=n_fig, num_epochs=10)
        metrics = {'train': {'monitor_values': {}, 'malignant_ap': [np.nan], 'benign_ap': [np.nan]},
                   'val': {'monitor_values': {}, 'malignant_ap': [np.nan], 'benign_ap': [np.nan]}}
        epochs = []
        for e in range(1, 4):
            for k in ('train', 'val'):
                metrics[k]['monitor_values'][e] = [{'loss': float(rs.rand() * 2), 'class_loss': float(rs.rand())} for _ in range(3)]
                metrics[k]['malignant_ap'].append(float(rs.rand()) if e != 2 else None)
                metrics[k]['benign_ap'].append(float(rs.rand()))
            epochs.append((e, copy.deepcopy(metrics)))
        out.append(dict(cf=cf.__dict__, epochs=epochs))
    return out


def main(ref_root):
    _make_stub()
    spec = importlib.util.spec_from_file_location('ref_plotting', os.path.join(ref_root, 'plotting.py'))
    plotting = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(plotting)
    golden = {'batch': [], 'hist': [], 'stat': [], 'monitor': []}

    def record(kind, case, fn):
        _REC.saved = []
        try:
            fn()
            golden[kind].append({'case': case, 'figures': _REC.saved})
        except Exception as e:       # the reference's own failure is part of what is recorded
            golden[kind].append({'case': case, 'figures': _REC.saved, 'raises': type(e).__name__})

    for args in ((2, 3, 1, 24, 20, None, 3, 1), (2, 2, 2, 18, 22, None, 2, 2, True), (3, 2, 1, 24, 20, 16, 3, 3),
                 (3, 3, 2, 16, 18, 12, 2, 4, False, (0, 1, 2)), (3, 2, 1, 16, 16, 6, 3, 5, True, (0, 1))):
        case = batch_case(*args)
        record('batch', case, lambda: run_batch(plotting, case))
    for case in hist_cases():
        record('hist', case, lambda: plotting.plot_prediction_hist(**case))
    for case in stat_cases():
        record('stat', case, lambda: plotting.plot_stat_curves(**case))
    for case in monitor_cases():
        def run():
            tp = plotting.TrainingPlot_2Panel(CF(**case['cf']))
            for e, m in case['epochs']:
                tp.update_and_save(m, e)
        record('monitor', case, run)
    with gzip.open(OUT, 'wb') as f:
        pickle.dump(golden, f, protocol=4)
    print('wrote', OUT, sum(len(v) for v in golden.values()), 'cases')


if __name__ == '__main__':
    main(sys.argv[1])
