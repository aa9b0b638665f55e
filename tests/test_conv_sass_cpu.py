"""What ptxas makes of the tensor-core conv kernels (conv3d_tc.cu, conv3d_tc_wgrad.cu), checked on the compiler's output (no GPU needed).

* No instantiation of conv_tc_kernel or conv_tc_wgrad_kernel gets a compiler-injected warpgroup fence (ptxas note C7519): a fence in front
  of an MMA makes it wait for the registers of the MMAs before it, so the batch of a stage no longer issues back to back.
* None of them spills, and the fprop/dgrad kernels of the full-resolution layers keep their residency: 288 threads per CTA, 3 CTAs per SM
  up to 72 registers (NT 32 and 48: the 18- and 36-channel layers), 2 CTAs per SM up to 112 (NT 64).
* The fixed-shape instantiations the Retina U-Net train step runs issue each stage (fprop/dgrad) or unit (wgrad) as one run of HGMMAs:
  one WARPGROUP.ARRIVE in front, no branch, fence or wait inside, scoreboard (gsb0) only on the last, and (fprop/dgrad) the accumulator
  overwritten by the first MMA instead of a run-time flag.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "medicaldetectiontoolkit_b200", "csrc")
SOURCES = ("conv3d_tc", "conv3d_tc_wgrad")
KERNELS = ("conv_tc_kernel", "conv_tc_wgrad_kernel")


def _tool(name):
    path = shutil.which(name)
    if path is None and os.path.exists(os.path.join("/usr/local/cuda/bin", name)):
        path = os.path.join("/usr/local/cuda/bin", name)
    return path


NVCC, CUOBJDUMP = _tool("nvcc"), _tool("cuobjdump")
pytestmark = pytest.mark.skipif(NVCC is None or CUOBJDUMP is None, reason="needs nvcc and cuobjdump (CUDA toolkit)")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{source: (ptxas -v log, object path)}, compiled with the flags of csrc/Makefile"""
    out = tmp_path_factory.mktemp("sass")
    procs = {}
    for src in SOURCES:
        obj = str(out / (src + ".o"))
        cmd = [NVCC, "-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
               "-Xptxas", "-v", "-I" + os.path.join(ROOT, "include"), "-c", os.path.join(CSRC, src + ".cu"), "-o", obj]
        procs[src] = (subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), obj)
    res = {}
    for src, (proc, obj) in procs.items():
        log = proc.communicate()[0]
        assert proc.returncode == 0, log[-4000:]
        res[src] = (log, obj)
    return res


def _ptxas_info(log):
    """{mangled kernel: {"regs": n, "spill": bytes stored + loaded, "c7519": notes}} for the two conv kernels"""
    info, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"\(C7519\).*in function '(\S+)'", line)
        if m:
            info.setdefault(m.group(1), {}).setdefault("c7519", 0)
            info[m.group(1)]["c7519"] += 1
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            info.setdefault(cur, {})["spill"] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            info.setdefault(cur, {})["regs"] = int(m.group(1))
    return {k: v for k, v in info.items() if any(("%d%s" % (len(n), n)) in k for n in KERNELS)}


def _all_info(compiled):
    info = {}
    for log, _ in compiled.values():
        info.update(_ptxas_info(log))
    return info


def _nt(name):
    """template arguments of a conv kernel's mangled name"""
    return [int(v) for v in re.findall(r"Li(\d+)E", name)]


def test_no_injected_fence_and_no_spill(compiled):
    info = _all_info(compiled)
    assert sum("conv_tc_kernel" in k for k in info) >= 8 and sum("conv_tc_wgrad_kernel" in k for k in info) >= 16, sorted(info)
    fenced = {k: v["c7519"] for k, v in info.items() if v.get("c7519")}
    assert not fenced, fenced
    spilled = {k: v["spill"] for k, v in info.items() if v.get("spill")}
    assert not spilled, spilled


def test_fprop_dgrad_residency(compiled):
    """3 CTAs of 288 threads per SM need <= 72 registers (65536 / (3 * 288) rounded down to the allocation granule), 2 CTAs <= 112"""
    info = _ptxas_info(compiled["conv3d_tc"][0])
    ceilings = {32: 72, 48: 72, 64: 112}
    checked = 0
    for name, v in info.items():
        nt = _nt(name)[0]
        if nt in ceilings:
            assert v["regs"] <= ceilings[nt], (name, v["regs"])
            checked += 1
    assert checked >= 3 + 2 * 10, checked   # the run-time-shaped kernels and the fixed shapes at both precisions


def _sass_functions(obj):
    text = subprocess.run([CUOBJDUMP, "-sass", obj], check=True, stdout=subprocess.PIPE, text=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", line)
        if cur is not None and m:
            funcs[cur].append(m.group(1).strip())
    return funcs


def _one_batch(instrs, n_mma):
    """the function's HGMMAs form one straight run of n_mma behind one WARPGROUP.ARRIVE; returns the run"""
    idx = [i for i, s in enumerate(instrs) if "HGMMA" in s]
    assert len(idx) == n_mma, (len(idx), n_mma)
    run = instrs[idx[0]:idx[-1] + 1]
    for s in run:
        assert not re.search(r"\bBRA\b|WARPGROUP|BAR|WARPSYNC|EXIT|RET", s), s
    assert sum("WARPGROUP.ARRIVE" in s for s in instrs) == 1
    arrive = max(i for i, s in enumerate(instrs[:idx[0]]) if "WARPGROUP.ARRIVE" in s)
    assert not any(re.search(r"\bBRA\b", s) for s in instrs[arrive:idx[0]]), instrs[arrive:idx[0]]
    hg = [instrs[i] for i in idx]
    assert "gsb0" in hg[-1] and not any("gsb0" in s for s in hg[:-1]), hg
    return hg


# (NT, planes, K steps, taps per stage): the 18-channel 3x3x3 and 7x7x7 layers, the 36-channel layers, the 64-channel heads
FPROP_BATCHES = [(32, 2, 2, 3), (32, 2, 2, 7), (48, 2, 4, 3), (48, 2, 4, 1), (64, 2, 4, 3), (64, 2, 4, 1), (48, 1, 4, 3)]
# (NC, planes, mtrick, K steps, dy swizzle, x swizzle)
WGRAD_BATCHES = [(96, 2, 1, 8, 64, 64), (224, 2, 1, 8, 64, 64), (192, 2, 1, 8, 128, 128), (192, 2, 1, 4, 128, 128), (64, 2, 0, 4, 128, 128)]


@pytest.mark.parametrize("shape", FPROP_BATCHES, ids=lambda s: "NT%d_planes%d_ksteps%d_tps%d" % s)
def test_fprop_dgrad_stage_is_one_batch(compiled, shape):
    nt, planes, ksteps, tps = shape
    name = "_ZN3mdt14conv_tc_kernelILi%dELi%dELi%dELi%dEEE" % shape
    funcs = _sass_functions(compiled["conv3d_tc"][1])
    fn = [k for k in funcs if k.startswith(name)]
    assert len(fn) == 1, (name, sorted(funcs))
    hg = _one_batch(funcs[fn[0]], tps * ksteps * (3 if planes == 2 else 1))
    assert all("64x%dx16" % nt in s for s in hg), hg[0]
    # scale_d = 0 on the first MMA only: the accumulator input is RZ with the predicate !UPT, the others accumulate
    assert re.search(r",\s*RZ\s*,\s*!UPT", hg[0]), hg[0]
    assert not any("RZ" in s for s in hg[1:]), hg


@pytest.mark.parametrize("shape", WGRAD_BATCHES, ids=lambda s: "NC%d_planes%d_mtrick%d_ksteps%d_swy%d_swx%d" % s)
def test_wgrad_unit_is_one_batch(compiled, shape):
    nc, planes, mtrick, ksteps, _, _ = shape
    name = "_ZN3mdt20conv_tc_wgrad_kernelILi%dELi%dELi%dELi%dELi%dELi%dEEE" % shape
    funcs = _sass_functions(compiled["conv3d_tc_wgrad"][1])
    fn = [k for k in funcs if k.startswith(name)]
    assert len(fn) == 1, (name, sorted(funcs))
    hg = _one_batch(funcs[fn[0]], ksteps * (1 if planes == 1 else 2 if mtrick else 3))
    assert all("64x%dx16" % nc in s for s in hg), hg[0]
