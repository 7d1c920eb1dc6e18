"""The C-ABI shared library loads on a machine without a GPU, exports every symbol declared in
include/jiminy_b200.h, and refuses (loudly) to create a batch when no CUDA device exists."""
import ctypes as C
import os
import re

import pytest

from jiminy_b200 import core, robots as R

from conftest import ROOT, has_cuda


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "jiminy_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(jb_[a-z_0-9]+)\s*\(", text)))


def test_header_symbols_exported():
    import __graft_entry__ as g
    g.build_cuda()
    lib = C.CDLL(core.library_path())
    names = _declared_symbols()
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert sorted(core.Api.SYMBOLS) == names      # the Python binding covers the whole header
    api = core.api()
    assert b"sm_90a" in api.dll.jb_version()


def test_default_options_match_reference_defaults():
    from jiminy_b200._ctypes_abi import JbOptions
    o = JbOptions()
    core.api().dll.jb_default_options(C.byref(o))
    assert (o.ode_solver, o.dt_max, o.tol_abs, o.tol_rel) == (2, 0.02, 1e-5, 1e-4)      # engine.h:318-339
    assert (o.contact_stiffness, o.contact_damping, o.contact_friction) == (1e6, 2e3, 1.0)
    assert o.contact_transition_eps == 1e-3 and o.contact_transition_velocity == 1e-2 and o.gravity[2] == -9.81


def test_planner_runs_without_device():
    robot, _ = R.load_robot("anymal")
    text, lanes = core.plan_describe(robot)
    assert "lanes=4" in text


@pytest.mark.skipif(has_cuda(), reason="only meaningful on a machine without a GPU")
def test_no_cpu_fallback():
    robot, opt = R.load_robot("cartpole")
    with pytest.raises(core.CudaUnavailable):
        core.BatchedEngine(robot, R.baseline_options("cartpole", opt), 4)


def test_unsupported_options_are_rejected():
    robot, opt = R.load_robot("anymal")
    opt["contacts"]["model"] = "impulse"
    with pytest.raises(ValueError):
        core.BatchedEngine(robot, opt, 1)
    opt["contacts"]["model"] = "constraint"
    opt["constraints"]["solver"] = "other"
    with pytest.raises(ValueError):
        core.BatchedEngine(robot, opt, 1)
