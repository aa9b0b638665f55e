#!/usr/bin/env python
"""Exact weight gradients of the tensor-core wgrad kernel (conv3d_tc_wgrad.cu) on seeded inputs, for tests/test_conv_wgrad_bits_gpu.py.

The kernel cuts each (column block, M tile) accumulation into chains of output lines, one per split, and wgrad_reduce_kernel adds the
partial sums in a fixed order; in ksplit mode the two warpgroups take alternate lines of a chain.  So dw is bit-reproducible, and any
change to which lines a chain holds, the order in which they are added, the warpgroup parity of a line or the order of the reduce shows
up in its last bits.  The file pins those bits.  The split count follows the SM count (wg_splits), so the bits hold for one SM count,
recorded with them.

CASES: the Retina U-Net's three full-resolution layers and its two head-conv levels at their train-step shapes, and small shapes for the
edges of the work decomposition: (column block, split, M tile) item counts that are not a multiple of the SM count, fewer items than SMs,
ksplit chains with an odd number of lines, two M tiles, and single-pass bf16.  To keep the file small, the larger cases store every
step-th output channel only: those rows still fall in every warp of the M tile, and every column block and input channel is kept.

Run on the H100 with the library to pin:  python tests/golden/make_wgrad_bits_golden.py [out.npz]  ->  tests/golden/wgrad_bits.npz"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from _guarded import _run_guarded  # noqa: E402
from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402

DEV = "cuda:0"
ALGO_TC = 2

# name: (n, cin, cout, kernel, stride, padding, spatial, precision, stored output channels co::step)
CASES = {
    "c0_18": (2, 18, 18, 3, 1, 1, (128, 128, 128), 0, 1),
    "c1_k7": (2, 18, 18, 7, (2, 2, 1), 3, (128, 128, 128), 0, 4),
    "p0_36": (2, 36, 36, 3, 1, 1, (128, 128, 128), 0, 2),
    "head64": (2, 64, 64, 3, 1, 1, (32, 32, 128), 0, 8),
    "head64_p3": (2, 64, 64, 3, 1, 1, (16, 16, 64), 0, 8),
    "ksplit_odd_chains": (2, 18, 18, 3, 1, 1, (16, 16, 128), 0, 1),   # 512 lines over 29 splits: chains of 17 and 18 lines
    "k7_odd_chains": (1, 18, 18, 7, (2, 2, 1), 3, (18, 22, 128), 0, 4),
    "few_items": (1, 36, 36, 3, 1, 1, (2, 2, 16), 0, 2),             # 4 lines: 36 items, fewer than SMs
    "two_mtiles": (1, 32, 160, 3, 1, 1, (8, 8, 64), 0, 8),
    "ksplit_bf16": (2, 18, 18, 3, 1, 1, (16, 16, 128), 1, 1),
}


def _triple(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v, v)


def desc(case):
    n, cin, cout, k, s, p, sp, prec, _ = CASES[case]
    return L.Conv3dDesc(n, *sp, cin, cout, *_triple(k), *_triple(s), *_triple(p), 0, prec, ALGO_TC)


def operands(case, seed):
    """(x, dy) as NDHWC fp32 on the device, drawn on the host from torch's CPU generator"""
    n, cin, cout, k, s, p, sp, _, _ = CASES[case]
    osp = tuple((i + 2 * pp - kk) // ss + 1 for i, kk, ss, pp in zip(sp, _triple(k), _triple(s), _triple(p)))
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, *sp, cin), generator=g)
    dy = torch.randn((n, *osp, cout), generator=g)
    return x.to(DEV), dy.to(DEV)


def wgrad(case, seed):
    """dw [cout, cin, kd, kh, kw] of mdt_conv3d_wgrad on the tensor cores, through guarded exact-size buffers; every guarded run (poisoned
    and zeroed workspace, three base offsets) must give the same bits"""
    n, cin, cout, k, _, _, _, _, _ = CASES[case]
    lib, d = L.load(), desc(case)
    assert lib.mdt_conv3d_algo(d, 2) == ALGO_TC, case
    x, dy = operands(case, seed)
    wshape = (cout, cin) + _triple(k)
    nws = lib.mdt_conv3d_workspace_bytes(d, 2)
    out = _run_guarded(lambda o, ws: lib.mdt_conv3d_wgrad(d, L.ptr(x), L.ptr(dy), o[0], o[1], ws, nws, L.stream_ptr()),
                       [int(np.prod(wshape)) * 4, cout * 4], nws)
    dw = out[0].view(torch.float32).view(wshape)
    assert bool(torch.isfinite(dw).all()), case
    return dw


def stored(case, dw):
    return dw[::CASES[case][8]].contiguous()


def seed_of(case):
    return 1000 + sorted(CASES).index(case)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "wgrad_bits.npz")
    res = {"num_sms": np.int64(torch.cuda.get_device_properties(0).multi_processor_count)}
    for case in CASES:
        res[case] = stored(case, wgrad(case, seed_of(case))).cpu().numpy()
        print(case, res[case].shape, flush=True)
    np.savez_compressed(out, **res)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
