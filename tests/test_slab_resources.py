"""CPU: the slab build's kernels keep the residency their grids are sized for, in the built library (cuobjdump
-res-usage).  The chunk grid and the slab count in Plan::layout assume 2 CTAs of 512 threads per SM for every fp32
slab kernel.  An fp32 instantiation whose registers x 512 threads no longer fit 2 CTAs in the 64 K registers of an
SM, or any slab kernel that spills, fails here instead of quietly halving the build's occupancy."""
import importlib.util
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "point-cloud-utils_b200", "libpcu_b200.so")
THREADS = 512      # kSlabThreads
CTAS = 2           # CTAs per SM the plan assumes for every fp32 slab kernel
REGS_PER_SM = 64 * 1024
_NAME = re.compile(r"(slab_hist|slab_partition|slab_sort)_kernelI([fd])NS_9Clouds(Val|Ptr)I[fd]EEEEvT0_")


def cuobjdump():
    spec = importlib.util.spec_from_file_location("sweep_sass", os.path.join(ROOT, "tools", "sweep_sass.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.cuobjdump()


def slab_usage(tool):
    """{(kernel, 'f' | 'd', 'Val' | 'Ptr'): {'REG': .., 'STACK': .., 'LOCAL': ..}} of the slab kernels."""
    text = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    out, key = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function\s+(\S+?):?\s*$", line)
        if m:
            n = _NAME.search(m.group(1))
            key = n.groups() if n else None
        elif key is not None and "REG:" in line:
            out[key] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            key = None
    return out


def test_slab_kernels_keep_their_ctas_per_sm(pcu):
    tool = cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump is not available")
    usage = slab_usage(tool)
    assert len(usage) == 12, sorted(usage)
    for (kernel, t, cs), u in sorted(usage.items()):
        assert u["STACK"] == 0 and u["LOCAL"] == 0, (kernel, t, cs, u)
        if t == "f":
            assert u["REG"] * THREADS * CTAS <= REGS_PER_SM, (kernel, cs, u["REG"])
