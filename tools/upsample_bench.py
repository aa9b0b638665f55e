"""The 2D decoder's bilinear x2 up-sampling on the library (mdt_upsample_linear2x_*, a fixed-order gather backward) against torch's
F.interpolate (CUDA kernels whose backward adds with float atomics), at the lidc 2D decoder shapes, and a 2D Retina U-Net train step with
each of the two paths.

    python tools/upsample_bench.py [--iters 20] [--steps 6] [--warmup 2] [--out result.json]

Ops: batch 20, end_filts 192, P2 72^2 -> P1 144^2 and P1 144^2 -> P0 288^2 (the P0 map alone is 1.27 GB), channels-last fp32.  Each op is
timed with CUDA events over --iters launches after warm-up; GB/s counts one read of the input and one write of the output.  The library's
and torch's fp32 results are compared with fp64 F.interpolate (max |err| / max |ref|) and with each other (largest ulp difference of the
results, and in ulps of the same op on |x|).
Step: make_cf('retina_unet', 2, (288, 288), exp='lidc_exp', batch_size=20), train_forward + backward + Adam, host clock around work that
ends in a device synchronise; the two paths alternate twice (lib, torch, lib, torch) so the spread between repeats is visible.
Prints one JSON line, with the card's name, power limit and SM clocks read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from medicaldetectiontoolkit_b200 import _lib as L  # noqa: E402
from medicaldetectiontoolkit_b200 import backbone as B  # noqa: E402

SHAPES = {"P2->P1": (20, 192, 72, 72), "P1->P0": (20, 192, 144, 144)}


def _events_ms(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _max_ulp(a, b):
    """largest distance in units in the last place between two fp32 tensors (finite, ordered as integers)"""
    ia, ib = a.contiguous().view(torch.int32).long(), b.contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


def _rel(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max())


def op_bench(iters):
    lib = L.load()
    out = {}
    for name, (n, c, h, w) in SHAPES.items():
        torch.manual_seed(0)
        x = torch.randn(n, c, h, w, device="cuda").contiguous(memory_format=torch.channels_last)
        gy = torch.randn(n, c, 2 * h, 2 * w, device="cuda").contiguous(memory_format=torch.channels_last)
        y = torch.empty_like(gy)
        gx = torch.empty_like(x)
        sp = L.stream_ptr()
        lib_f = lambda: L.check(lib.mdt_upsample_linear2x_forward(L.ptr(x), L.ptr(y), n, h, w, 1, c, sp))   # noqa: E731
        lib_b = lambda: L.check(lib.mdt_upsample_linear2x_backward(L.ptr(gy), L.ptr(gx), n, h, w, 1, c, sp))   # noqa: E731
        torch_f = lambda: torch.ops.aten.upsample_bilinear2d(x, [2 * h, 2 * w], False, 2.0, 2.0)   # noqa: E731
        torch_b = lambda: torch.ops.aten.upsample_bilinear2d_backward(gy, [2 * h, 2 * w], [n, c, h, w], False, 2.0, 2.0)   # noqa: E731
        nbytes = 4 * (x.numel() + gy.numel())
        r = {"x": [n, c, h, w], "y": [n, c, 2 * h, 2 * w], "y_GB": round(4 * gy.numel() / 1e9, 3)}
        for tag, fn in (("lib_fwd", lib_f), ("torch_fwd", torch_f), ("lib_bwd", lib_b), ("torch_bwd", torch_b)):
            ms = _events_ms(fn, iters)
            r[tag + "_ms"] = round(ms, 4)
            r[tag + "_GBps"] = round(nbytes / ms / 1e6, 1)
        # accuracy on the same inputs: fp64 reference per batch item (keeps the fp64 copies small)
        lib_f()
        lib_b()
        yt, gxt = torch_f(), torch_b()
        torch.cuda.synchronize()
        r["fwd_max_ulp_lib_vs_torch"] = _max_ulp(y, yt)
        # the same difference in ulps of the magnitude (the op on |x|): an output is a convex combination, so where its terms cancel an
        # rounding-level difference is many ulps of the (small) result but a fraction of an ulp of the terms
        xa, ya = x.abs(), torch.empty_like(y)
        L.check(lib.mdt_upsample_linear2x_forward(L.ptr(xa), L.ptr(ya), n, h, w, 1, c, sp))
        _, e = torch.frexp(ya)
        r["fwd_max_diff_in_ulps_of_magnitude"] = float(((y - yt).abs() / torch.ldexp(torch.ones_like(ya), e - 24)).max())
        del xa, ya, e
        r["fwd_equal_lib_vs_torch_fraction"] = float((y == yt).double().mean())
        e = {"fwd_lib": 0.0, "fwd_torch": 0.0, "bwd_lib": 0.0, "bwd_torch": 0.0}
        for b in range(0, n, 4):
            x64 = x[b:b + 4].double().requires_grad_(True)
            ref = F.interpolate(x64, scale_factor=2, mode="bilinear", align_corners=False)
            ref.backward(gy[b:b + 4].double())
            e["fwd_lib"] = max(e["fwd_lib"], _rel(y[b:b + 4], ref.detach()))
            e["fwd_torch"] = max(e["fwd_torch"], _rel(yt[b:b + 4], ref.detach()))
            e["bwd_lib"] = max(e["bwd_lib"], _rel(gx[b:b + 4], x64.grad))
            e["bwd_torch"] = max(e["bwd_torch"], _rel(gxt[b:b + 4], x64.grad))
            del x64, ref
        r["max_err_over_max_ref_vs_fp64"] = {k: float("%.3g" % v) for k, v in e.items()}
        lib_b()
        g2 = gx.clone()
        lib_b()
        torch.cuda.synchronize()
        r["lib_bwd_repeat_bit_identical"] = bool(torch.equal(g2, gx))
        r["torch_bwd_repeat_bit_identical"] = bool(torch.equal(torch_b(), gxt))
        out[name] = r
        del x, gy, y, gx, yt, gxt, g2
        torch.cuda.empty_cache()
    return out


def step_bench(steps, warmup):
    from medicaldetectiontoolkit_b200 import retina_unet
    from medicaldetectiontoolkit_b200.configs import make_cf, synthetic_batch
    cf = make_cf('retina_unet', 2, (288, 288), exp='lidc_exp', batch_size=20)
    torch.manual_seed(0)
    net = retina_unet.net(cf, None).cuda()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    batches = [synthetic_batch(cf, 20, seed=i) for i in range(2)]
    lib_forward = B.Interpolate.forward

    def torch_forward(self, x):
        return F.interpolate(x, scale_factor=self.scale_factor, mode=self.mode, align_corners=False)

    def run(path):
        B.Interpolate.forward = lib_forward if path == "lib" else torch_forward
        try:
            net.load_state_dict(state)
            opt = torch.optim.Adam(net.parameters(), lr=1e-4)
            times = []
            for i in range(warmup + steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                net.zero_grad(set_to_none=True)
                res = net.train_forward(batches[i % 2])
                res['torch_loss'].backward()
                opt.step()
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            t = sorted(times[warmup:])
            return {"median_ms": round(1e3 * t[len(t) // 2], 1), "min_ms": round(1e3 * t[0], 1), "max_ms": round(1e3 * t[-1], 1)}
        finally:
            B.Interpolate.forward = lib_forward
    out = {"shape": "retina_unet 2D lidc_exp, 20 x 1 x 288 x 288, end_filts %d" % cf.end_filts, "steps": steps, "warmup": warmup, "runs": []}
    for path in ("lib", "torch", "lib", "torch"):
        out["runs"].append(dict(path=path, **run(path)))
    out["peak_mem_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    return out


def _smi():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the query is informational
        return 'unavailable: %s' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--steps', type=int, default=6)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('upsample_bench: no CUDA device (the numbers are GPU timings; there is no CPU mode)')
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi_before": _smi(), "ops": op_bench(a.iters)}
    res["train_step"] = step_bench(a.steps, a.warmup)
    res["nvidia_smi_after"] = _smi()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
