"""CPU: the k = 1 sweep's candidate loop keeps its loads in flight in the built library (tools/sweep_sass.py reads
the SASS).  Every fp32 nn1_kernel instantiation must issue both candidate loads of a trip before the first
instruction that reads either, without spills or a stack frame, within the 40 registers of six CTAs per SM;
the fp64 ones must keep at least the loads in flight they have had."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_tool():
    spec = importlib.util.spec_from_file_location("sweep_sass", os.path.join(ROOT, "tools", "sweep_sass.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_nn1_candidate_loads_in_flight(pcu):
    tool = load_tool()
    if tool.cuobjdump() is None:
        pytest.skip("cuobjdump is not available")
    rows = tool.report()
    assert len(rows) == 8, [r["name"] for r in rows]
    for r in rows:
        assert r["stack"] == 0 and r["local"] == 0 and r["spill_insns"] == 0, r
        if r["name"].startswith("<float"):
            assert r["regs"] <= 40, r
            assert r["loads_in_flight"] >= 2, r
        else:   # one fp64 point is two 128-bit loads; the per-point path keeps both candidates in flight
            assert r["regs"] <= 64, r
            assert r["loads_in_flight"] >= (4 if "kOut=true" in r["name"] else 2), r
