"""Per-robot geometry without a GPU: the validity check and the configuration patch of the device headers (shared by the blocking
setter, the solve kernel and the emulator) against numpy restatements, the compiled per-robot-geometry solve kernels against their
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

import robot_geometry_cases as rg
from mpc_local_planner_b200 import capi, configs

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB = []


def _lib():
    """the emulator with the two functions exported (tests/robot_geometry/), compiled with the flags of emu/Makefile"""
    if not _LIB:
        out = os.path.join(tempfile.mkdtemp(prefix="mpcb200_robot_geometry_"), "robot_geometry_emu.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-march=x86-64-v3", "-fPIC", "-std=c++17", "-shared", "-o", out,
                               os.path.join(_HERE, "robot_geometry", "robot_geometry_emu.cpp"), "-lm"], stdout=subprocess.DEVNULL)
        lib = C.CDLL(out)
        lib.emu_robot_geometry_valid.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_geometry.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_geometry.restype = None
        _LIB.append(lib)
    return _LIB[0]


def _dp(r):
    return np.ascontiguousarray(r, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


def _valid(cfg, rec):
    r = np.ascontiguousarray(rec, dtype=np.float64)
    return bool(_lib().emu_robot_geometry_valid(C.byref(cfg), _dp(r)))


def _config(robot, footprint):
    """cfg 3 with the given robot and footprint type, each footprint with values of its own"""
    c = configs.cfg3()
    c.robot_type = robot
    c.length_rear, c.length_front = 0.2, 0.25
    c.footprint_type = footprint
    c.footprint_params[:] = {capi.FOOTPRINT_CIRCULAR: [0.25, 0, 0, 0], capi.FOOTPRINT_TWO_CIRCLES: [0.2, 0.18, 0.1, 0.15],
                             capi.FOOTPRINT_LINE: [0.25, 0.05, -0.1, -0.05]}.get(footprint, [0.0, 0.0, 0.0, 0.0])
    return c


_TYPES = list(itertools.product(range(4), range(5)))


def _words_read(cfg):
    """the record words the handle's robot and footprint types read"""
    w = []
    if cfg.robot_type in rg.CARS:
        w.append(capi.GEO_WHEELBASE)
    elif cfg.robot_type == capi.ROBOT_KIN_BICYCLE:
        w += [capi.GEO_LENGTH_REAR, capi.GEO_LENGTH_FRONT]
    if cfg.footprint_type == capi.FOOTPRINT_CIRCULAR:
        w.append(rg.FP)
    elif cfg.footprint_type in (capi.FOOTPRINT_TWO_CIRCLES, capi.FOOTPRINT_LINE):
        w += list(range(rg.FP, rg.FP + 4))
    elif cfg.footprint_type == capi.FOOTPRINT_POLYGON:
        w += [rg.NP] + list(range(rg.XY, rg.XY + 2 * cfg.n_poly))
    return w


@pytest.mark.parametrize("robot,footprint", _TYPES)
def test_validity_matches_the_rules(robot, footprint):
    cfg = _config(robot, footprint)
    base = rg.record_of(cfg)
    assert _valid(cfg, base) and rg.rule(cfg, base)
    specials = [np.nan, np.inf, -np.inf, 0.0, -0.0, -1e-300, -0.3, 1e300]
    for w, v in itertools.product(range(rg.W), specials):   # one special value in each word
        r = base.copy(); r[w] = v
        assert _valid(cfg, r) == rg.rule(cfg, r), f"word {w} = {v}"
    unread = [w for w in range(rg.W) if w not in _words_read(cfg)]
    r = base.copy(); r[unread] = np.nan   # words the handle does not read may hold anything
    assert _valid(cfg, r)
    if footprint == capi.FOOTPRINT_POLYGON:
        for n in (0.0, 0.5, 1.0, 2.5, 3.0, 7.0 + 1e-9, 16.0, 16.5, 17.0, -1.0, -0.0, 1e300, np.inf, -np.inf, np.nan):
            r = base.copy(); r[rg.NP] = n
            assert _valid(cfg, r) == rg.rule(cfg, r), f"n_poly = {n}"
        for n in range(1, capi.MAX_POLY + 1):   # n_poly vertices finite, the rest NaN
            r = base.copy(); r[rg.NP] = n; r[rg.XY:] = np.nan; r[rg.XY:rg.XY + 2 * n] = 0.1
            assert _valid(cfg, r)
            if n < capi.MAX_POLY:
                r[rg.XY + 2 * n - 1] = np.nan
                assert not _valid(cfg, r)
    rng = np.random.default_rng(robot * 5 + footprint)
    pool = np.array([np.nan, np.inf, -np.inf, -1.0, -0.0, 0.0, 0.2, 3.0, 17.0, 2.5])
    for _ in range(3000):   # random records: words scaled, signs flipped, special values, in every combination
        r = base * rng.uniform(-0.5, 1.5, rg.W)
        r[rg.NP] = rng.integers(-1, 19)
        hit = rng.random(rg.W) < 0.1
        r[hit] = rng.choice(pool, hit.sum())
        assert _valid(cfg, r) == rg.rule(cfg, r), f"{r}"


@pytest.mark.parametrize("robot,footprint", _TYPES)
def test_patch_sets_exactly_the_fields_read(robot, footprint):
    cfg = _config(robot, footprint)
    rng = np.random.default_rng(40 + robot * 5 + footprint)
    for _ in range(20):
        rec = rng.uniform(0.1, 3.0, rg.W)
        rec[rg.NP] = rng.integers(1, capi.MAX_POLY + 1)
        got = cfg.copy()
        _lib().emu_apply_robot_geometry(C.byref(got), _dp(rec))
        want = rg.with_geometry(cfg, rec)
        assert C.string_at(C.addressof(got), C.sizeof(got)) == C.string_at(C.addressof(want), C.sizeof(want))


# ---- the per-robot-geometry solve kernels: -Xptxas -v lines and occupancy ----
_ENTRY = re.compile(r"Compiling entry function '(_Z\d+solve_fused(?:_fleet)?_kernel\w+)' for 'sm_90a'\n"
                    r"ptxas info\s+: Function properties for \1\n(.*)\n(ptxas info\s+: Used .*)")
_USED = re.compile(r"Used (\d+) registers, .* (\d+) bytes smem")
_FLEET = "solve_fused_fleet_kernel"


def _entries(text):
    """{kernel: (stack / spill line, registers / smem line)} of the solve kernels in -Xptxas -v output"""
    return {m.group(1): (m.group(2).strip(), m.group(3).strip()) for m in _ENTRY.finditer(text)}


def _base_of(fleet_name):
    """the solve_fused_kernel instantiation a per-robot-geometry entry is the form of (same template arguments, two parameters
    fewer)"""
    return fleet_name.replace("24solve_fused_fleet_kernel", "18solve_fused_kernel").replace("9FusedArgs9RobotArgsPKd", "9FusedArgs")


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_fleet_kernels_ptxas_lines_and_occupancy(tmp_path):
    """Every solve_fused_fleet_kernel instantiation (the 16 MODEL_GENERIC variants): its -Xptxas -v lines as recorded in
    tests/golden/ptxas_solve_fused_fleet.txt, and the registers and shared memory of its base kernel -- so CUDA fits as many of its
    CTAs on an SM as of the base kernel's, for every image size."""
    import __graft_entry__ as g
    cmd = [g._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
           "-o", str(tmp_path / "k.cubin"), os.path.join(_ROOT, "mpc_local_planner_b200", "csrc", "mpcb200.cu")]
    now = _entries(subprocess.run(cmd, capture_output=True, text=True, check=True).stderr)
    fleet = {k: v for k, v in now.items() if _FLEET in k}
    with open(os.path.join(_HERE, "golden", "ptxas_solve_fused_fleet.txt")) as f:
        recorded = _entries(f.read())
    assert len(recorded) == 16 and fleet == recorded
    for k, (_, used) in fleet.items():
        base = now[_base_of(k)][1]
        assert _USED.search(used).groups() == _USED.search(base).groups(), f"{k}: {used} vs {base}"


# ---- the Python setters without a device ----
def test_geometry_symbols_are_exported():
    assert "mpcb200_set_robot_geometry" in capi.EXPORTS and "mpcb200_set_robot_geometry_async" in capi.EXPORTS
    lib = capi.load_library()
    lib.mpcb200_set_robot_geometry, lib.mpcb200_set_robot_geometry_async   # noqa: B018


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
    for bad in (np.zeros(rg.W), np.zeros((2, rg.W - 1)), np.zeros((2, rg.W + 1)), np.zeros((1, 2, rg.W))):
        with pytest.raises(ValueError):
            s.set_robot_geometry(bad)
    assert s.lib.calls == []
    s.set_robot_geometry(None)
    assert [c[0] for c in s.lib.calls] == ["mpcb200_set_robot_geometry"] and s.lib.calls[0][1][1] == 0
