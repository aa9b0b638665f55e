"""The tensor-core weight gradient (conv3d_tc_wgrad.cu) keeps its bits: dw of mdt_conv3d_wgrad on seeded inputs equals, bit for bit, the
dw recorded in tests/golden/wgrad_bits.npz (tests/golden/make_wgrad_bits_golden.py), at the Retina U-Net's full-resolution and head layers
and at the edges of the work decomposition.  Each call runs through guarded, poisoned exact-size buffers, several times, and every run must
give the same bits.  A change to the lines of a chain, their order, the warpgroup that takes a line in ksplit mode or the order of the
reduce changes the last bits of dw and fails here, even where it stays inside the tolerance of tests/test_conv_gpu.py."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_wgrad_bits_golden as WB  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "wgrad_bits.npz")) as f:
        gold = {k: f[k] for k in f.files}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != int(gold["num_sms"]):
        pytest.skip("the split-K cut follows the SM count: recorded on %d SMs, this device has %d" % (int(gold["num_sms"]), sms))
    return gold


@pytest.mark.parametrize("case", sorted(WB.CASES))
def test_wgrad_bits(golden, case):
    got = WB.stored(case, WB.wgrad(case, WB.seed_of(case))).cpu()
    want = torch.from_numpy(golden[case])
    assert got.shape == want.shape, (got.shape, want.shape)
    if not torch.equal(got, want):
        diff = (got != want)
        pytest.fail("%s: %d of %d elements differ, max |diff| %.3g" % (case, int(diff.sum()), diff.numel(), float((got - want).abs().max())))
