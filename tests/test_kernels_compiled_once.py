"""CPU: every kernel of the built library is compiled in exactly one translation unit, and the library exports none of
the functions its units share (namespace pcu_internal).  A kernel template instantiated, or a kernel defined in a
header included, by two units is compiled twice: the library grows, and the two copies can drift apart.  Shared
kernels are declared in a header and defined in one unit instead, as the record sort and mc_heads_kernel are in
runtime.cu."""
import collections
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "point-cloud-utils_b200", "libpcu_b200.so")


def cuobjdump():
    spec = importlib.util.spec_from_file_location("sweep_sass", os.path.join(ROOT, "tools", "sweep_sass.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.cuobjdump()


def test_every_kernel_is_compiled_once(pcu):
    tool = cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump is not available")
    text = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    names = [m.group(1) for m in re.finditer(r"^\s*Function\s+(\S+?):?\s*$", text, re.M)]
    assert names, "cuobjdump listed no kernels"
    twice = sorted(n for n, c in collections.Counter(names).items() if c > 1)
    assert not twice, twice


def test_no_internal_function_is_exported(pcu):
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm is not available")
    text = subprocess.run([nm, "-D", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    assert re.search(r"\bT pcu_b200_abi_version$", text, re.M), "the C entry points are missing"
    leaked = [line for line in text.splitlines() if "pcu_internal" in line]
    assert not leaked, leaked
