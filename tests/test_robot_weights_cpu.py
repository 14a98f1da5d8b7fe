"""Per-robot weights without a GPU: the validity check and the configuration patch of the device headers (shared by the blocking
setter, the solve kernel and the emulator) against numpy restatements, the compiled per-robot-weights solve kernels against their
recorded -Xptxas -v lines and the occupancy of the kernels they are a form of, and the Python setters' argument checks."""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import robot_weights_cases as rw
from mpc_local_planner_b200 import capi, configs

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB = []


def _lib():
    """the emulator with the two functions exported (tests/robot_weights/), compiled with the flags of emu/Makefile"""
    if not _LIB:
        out = os.path.join(tempfile.mkdtemp(prefix="mpcb200_robot_weights_"), "robot_weights_emu.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-march=x86-64-v3", "-fPIC", "-std=c++17", "-shared", "-o", out,
                               os.path.join(_HERE, "robot_weights", "robot_weights_emu.cpp"), "-lm"], stdout=subprocess.DEVNULL)
        lib = C.CDLL(out)
        lib.emu_robot_weights_valid.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_weights.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_weights.restype = None
        _LIB.append(lib)
    return _LIB[0]


def _dp(r):
    return np.ascontiguousarray(r, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


def _valid(cfg, rec):
    r = np.ascontiguousarray(rec, dtype=np.float64)
    return bool(_lib().emu_robot_weights_valid(C.byref(cfg), _dp(r)))


def _config(objective, terminal, hybrid, vp, xf_fixed):
    """cfg 2 with the given objective, terminal cost, hybrid flag (0 off; 1 on with zero Q, so the term is on; 2 on with the
    configuration's Q, so the reference falls back to the plain quadratic form), via-point attraction of the quadratic form and
    fixed final state; the via-point weights non-zero"""
    c = configs.cfg2()
    c.objective, c.terminal_cost, c.vp_attraction_with_quadratic = objective, terminal, vp
    c.variable_dt = int(objective != capi.OBJ_QUADRATIC_FORM or hybrid == 1)
    c.xf_fixed[:] = xf_fixed
    c.hybrid_cost_minimum_time = int(hybrid > 0)
    if hybrid == 1:
        c.Q[:] = [0.0] * 9
    c.vp_position_weight, c.vp_orientation_weight = 8.0, 0.5
    return c


_CASES = [(o, t, h, v, x) for o, t, h, v, x in itertools.product(
    (capi.OBJ_QUADRATIC_FORM, capi.OBJ_MINIMUM_TIME, capi.OBJ_MINIMUM_TIME_VIA_POINTS), (0, 1), (0, 1, 2), (0, 1),
    ((0, 0, 0), (1, 1, 0), (1, 1, 1)))
    if (o == capi.OBJ_QUADRATIC_FORM or (h, v) == (0, 0))]


def test_the_cases_cover_every_objective_and_a_handle_reading_nothing():
    cfgs = [_config(*k) for k in _CASES]
    assert {c.objective for c in cfgs} == {capi.OBJ_QUADRATIC_FORM, capi.OBJ_MINIMUM_TIME, capi.OBJ_MINIMUM_TIME_VIA_POINTS}
    hyb = [rw.hybrid(c, list(c.Q), list(c.R)) for c in cfgs]
    assert any(hyb) and any(c.hybrid_cost_minimum_time and not h for c, h in zip(cfgs, hyb))
    assert any(not rw.words_read(c) for c in cfgs) and any(rw.terminal(c) and not rw.quadratic(c) for c in cfgs)


@pytest.mark.parametrize("objective,terminal,hybrid,vp,xf_fixed", _CASES)
def test_validity_matches_the_rules(objective, terminal, hybrid, vp, xf_fixed):
    cfg = _config(objective, terminal, hybrid, vp, xf_fixed)
    base = rw.record_of(cfg)
    assert _valid(cfg, base) and rw.rule(cfg, base)
    specials = [np.nan, np.inf, -np.inf, 0.0, -0.0, -1e-300, -0.3, 1e300]
    for w, v in itertools.product(range(rw.W), specials):   # one special value in each word
        r = base.copy(); r[w] = v
        assert _valid(cfg, r) == rw.rule(cfg, r), f"word {w} = {v}"
    read = rw.words_read(cfg)
    r = base.copy(); r[[w for w in range(rw.W) if w not in read]] = np.nan   # words the handle does not read may hold anything
    assert _valid(cfg, r)
    for w in read:   # NaN and inf in any word that is read
        for v in (np.nan, np.inf, -np.inf):
            r = base.copy(); r[w] = v
            assert not _valid(cfg, r), f"word {w} = {v}"
    if rw.quadratic(cfg):   # the hybrid term: zero Q with non-zero R, switched on or off by the record
        for q, rr in ((0.0, 1.0), (0.0, 0.0), (1.0, 1.0), (-0.0, 1.0), (0.0, -0.0)):
            r = base.copy(); r[rw.Q:rw.Q + 9] = q; r[rw.R:rw.R + 4] = rr
            assert _valid(cfg, r) == rw.rule(cfg, r), f"Q = {q}, R = {rr}"
            assert _valid(cfg, r) == (rw.hybrid(cfg, r[rw.Q:rw.Q + 9], r[rw.R:rw.R + 4]) == rw.hybrid(cfg, list(cfg.Q), list(cfg.R)))
    if not read:   # a handle that reads no weight: every record passes the check (the setters refuse records there)
        assert _valid(cfg, np.full(rw.W, np.nan))
    rng = np.random.default_rng(_CASES.index((objective, terminal, hybrid, vp, xf_fixed)))
    pool = np.array([np.nan, np.inf, -np.inf, -1.0, -0.0, 0.0, 0.2, 3.0])
    for _ in range(2000):   # random records: words scaled, signs flipped, zero blocks, special values, in every combination
        r = base * rng.uniform(-0.5, 1.5, rw.W)
        if rng.random() < 0.3:
            r[rw.Q:rw.Q + 9] = 0.0
        if rng.random() < 0.2:
            r[rw.R:rw.R + 4] = 0.0
        hit = rng.random(rw.W) < 0.08
        r[hit] = rng.choice(pool, hit.sum())
        assert _valid(cfg, r) == rw.rule(cfg, r), f"{r}"


@pytest.mark.parametrize("objective,terminal,hybrid,vp,xf_fixed", _CASES)
def test_patch_sets_exactly_the_words_read(objective, terminal, hybrid, vp, xf_fixed):
    cfg = _config(objective, terminal, hybrid, vp, xf_fixed)
    rng = np.random.default_rng(7)
    for _ in range(20):
        rec = rng.uniform(0.1, 3.0, rw.W)
        got = cfg.copy()
        _lib().emu_apply_robot_weights(C.byref(got), _dp(rec))
        want = rw.with_weights(cfg, rec)
        assert C.string_at(C.addressof(got), C.sizeof(got)) == C.string_at(C.addressof(want), C.sizeof(want))


# ---- the per-robot-weights solve kernels: -Xptxas -v lines and occupancy ----
_ENTRY = re.compile(r"Compiling entry function '(_Z\d+solve_fused(?:_weights|_robot)?_kernel\w+)' for 'sm_90a'\n"
                    r"ptxas info\s+: Function properties for \1\n(.*)\n(ptxas info\s+: Used .*)")
_ANY_ENTRY = re.compile(r"Compiling entry function '(\w+)'")
_USED = re.compile(r"Used (\d+) registers, .* (\d+) bytes smem")
_WEIGHTS = "solve_fused_weights_kernel"


def _entries(text):
    """{kernel: (stack / spill line, registers / smem line)} of the solve kernels in -Xptxas -v output"""
    return {m.group(1): (m.group(2).strip(), m.group(3).strip()) for m in _ENTRY.finditer(text)}


def _robot_of(weights_name):
    """the solve_fused_robot_kernel instantiation with the same template arguments as a per-robot-weights entry (two parameters
    fewer)"""
    return weights_name.replace("26solve_fused_weights_kernel", "24solve_fused_robot_kernel").replace("9RobotArgsPKdS5_", "9RobotArgs")


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_weights_kernels_ptxas_lines_and_occupancy(tmp_path):
    """The translation unit of the per-robot-weights entries (mpcb200_weights.cu) compiles exactly the 28 solve_fused_weights_kernel
    instantiations, every one with its -Xptxas -v lines as recorded in tests/golden/ptxas_solve_fused_weights.txt and the
    registers and shared memory of the per-robot-limits entry of the same variant (tests/golden/ptxas_solve_fused_robot.txt, whose
    test holds those equal to the base solve_fused_kernel's) -- so CUDA fits as many of its CTAs on an SM as of the base kernel's,
    for every image size."""
    import __graft_entry__ as g
    cmd = [g._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
           "-o", str(tmp_path / "k.cubin"), os.path.join(_ROOT, "mpc_local_planner_b200", "csrc", "mpcb200_weights.cu")]
    text = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    weights = _entries(text)
    assert all(_WEIGHTS in k for k in _ANY_ENTRY.findall(text)) and len(_ANY_ENTRY.findall(text)) == len(weights)
    with open(os.path.join(_HERE, "golden", "ptxas_solve_fused_weights.txt")) as f:
        recorded = _entries(f.read())
    assert len(recorded) == 28 and weights == recorded
    with open(os.path.join(_HERE, "golden", "ptxas_solve_fused_robot.txt")) as f:
        robot = _entries(f.read())
    for k, (_, used) in weights.items():
        assert _USED.search(used).groups() == _USED.search(robot[_robot_of(k)][1]).groups(), f"{k}: {used} vs {robot[_robot_of(k)][1]}"


# ---- the Python setters without a device ----
def test_weights_symbols_are_exported():
    assert "mpcb200_set_robot_weights" in capi.EXPORTS and "mpcb200_set_robot_weights_async" in capi.EXPORTS
    lib = capi.load_library()
    lib.mpcb200_set_robot_weights, lib.mpcb200_set_robot_weights_async   # noqa: B018


class _NoCalls:
    """a library stand-in that records every call"""
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*a):
            self.calls.append((name, a))
            return 0
        return f


def test_setter_checks_the_shape_before_any_call():
    s = capi.BatchSolver.__new__(capi.BatchSolver)
    s.lib, s.h = _NoCalls(), None
    for bad in (np.zeros(rw.W), np.zeros((2, rw.W - 1)), np.zeros((2, rw.W + 1)), np.zeros((1, 2, rw.W))):
        with pytest.raises(ValueError):
            s.set_robot_weights(bad)
    assert s.lib.calls == []
    s.set_robot_weights(None)
    assert [c[0] for c in s.lib.calls] == ["mpcb200_set_robot_weights"] and s.lib.calls[0][1][1] == 0
