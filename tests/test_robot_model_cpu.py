"""Per-robot model without a GPU: the validity check and the configuration patch of the device headers (shared by the blocking
setters, the solve kernel and the emulator) against a numpy restatement, for every handle type pair and every record type pair,
the compiled per-robot-model solve kernels against their recorded -Xptxas -v lines and the occupancy of the kernels they are a
form of, and the Python setters' argument checks."""
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
import robot_model_cases as rm
from mpc_local_planner_b200 import capi, configs

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB = []


def _lib():
    """the emulator with the two functions exported (tests/robot_model/), compiled with the flags of emu/Makefile"""
    if not _LIB:
        out = os.path.join(tempfile.mkdtemp(prefix="mpcb200_robot_model_"), "robot_model_emu.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-march=x86-64-v3", "-fPIC", "-std=c++17", "-shared", "-o", out,
                               os.path.join(_HERE, "robot_model", "robot_model_emu.cpp"), "-lm"], stdout=subprocess.DEVNULL)
        lib = C.CDLL(out)
        lib.emu_robot_model_valid.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double), C.POINTER(C.c_double)]
        lib.emu_apply_robot_model.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_model.restype = None
        _LIB.append(lib)
    return _LIB[0]


def _dp(r):
    return np.ascontiguousarray(r, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


def _valid(cfg, rec, geo=None):
    r = np.ascontiguousarray(rec, dtype=np.float64)
    g = None if geo is None else np.ascontiguousarray(geo, dtype=np.float64)
    return bool(_lib().emu_robot_model_valid(C.byref(cfg), _dp(r), None if g is None else _dp(g)))


def _handle(robot, footprint, bare):
    """cfg 3 with the given types; `bare`: geometry values that only some types accept (no polygon vertices, a zero wheelbase,
    a negative radius and rear length), else values every type accepts"""
    c = configs.cfg3()
    c.robot_type, c.footprint_type = robot, footprint
    c.length_rear, c.length_front = 0.2, 0.25
    c.footprint_params[:] = [0.25, 0.18, 0.1, 0.15]
    if bare:
        c.n_poly, c.wheelbase, c.length_rear = 0, 0.0, -0.2
        c.footprint_params[:] = [-0.25, 0.18, 0.1, 0.15]
        for i in range(2 * capi.MAX_POLY):
            c.poly_xy[i] = 0.0
    return c


def _geometry_for(robot, footprint, rng, nan_unread=True):
    """a geometry record valid for the types, the words those types do not read NaN"""
    r = np.full(rg.W, np.nan) if nan_unread else np.zeros(rg.W)
    if robot in rg.CARS:
        r[capi.GEO_WHEELBASE] = rng.uniform(0.3, 0.6)
    elif robot == capi.ROBOT_KIN_BICYCLE:
        r[capi.GEO_LENGTH_REAR], r[capi.GEO_LENGTH_FRONT] = rng.uniform(0.1, 0.3), rng.uniform(0.0, 0.3)
    if footprint == capi.FOOTPRINT_CIRCULAR:
        r[rg.FP] = rng.uniform(0.1, 0.4)
    elif footprint in (capi.FOOTPRINT_TWO_CIRCLES, capi.FOOTPRINT_LINE):
        r[rg.FP:rg.FP + 4] = rng.uniform(0.05, 0.3, 4)
    elif footprint == capi.FOOTPRINT_POLYGON:
        n = int(rng.integers(3, 17))
        r[rg.NP] = n
        r[rg.XY:rg.XY + 2 * n] = rg.polygon(n, rng).ravel()
    return r


_SPECIALS = [np.nan, np.inf, -np.inf, -0.0, 0.0, 0.5, 2.5, 3.0, 4.0, 5.0, -1.0, 1e300, -1e-300, 2.0000000000000004]


@pytest.mark.parametrize("robot,footprint", rm.TYPES)
@pytest.mark.parametrize("bare", [False, True])
def test_validity_matches_the_rule(robot, footprint, bare):
    """every record type pair on this handle type pair, with the configuration's geometry and with a geometry record of each
    type pair (its unread words NaN), and special values in both words"""
    cfg = _handle(robot, footprint, bare)
    rng = np.random.default_rng(robot * 5 + footprint + 20 * bare)
    geos = {t: _geometry_for(*t, rng) for t in rm.TYPES}
    for t in rm.TYPES:
        rec = rm.record(*t)
        assert _valid(cfg, rec) == rm.rule(cfg, rec), f"record {t}"
        if not bare:
            assert _valid(cfg, rec)   # values every type accepts
        for tg, g in geos.items():   # a geometry record valid for its own types: valid for a record of other types only by its words
            assert _valid(cfg, rec, g) == rm.rule(cfg, rec, g), f"record {t} geometry for {tg}"
            if tg == t:
                assert _valid(cfg, rec, g)
    for w, v in itertools.product(range(rm.W), _SPECIALS):   # one special value in one word of a record of the handle's types
        rec = rm.record_of(cfg); rec[w] = v
        g = geos[(robot, footprint)]
        assert _valid(cfg, rec) == rm.rule(cfg, rec), f"word {w} = {v}"
        assert _valid(cfg, rec, g) == rm.rule(cfg, rec, g), f"word {w} = {v} with a geometry record"
        hi = 3 if w == rm.RT else 4
        if not (np.isfinite(v) and 0 <= v <= hi and v == np.floor(v)):
            assert not _valid(cfg, rec, g), f"word {w} = {v}"
    for v in (-0.0, 0.0):   # -0 is 0
        rec = rm.record(v, v)
        assert _valid(cfg, rec, geos[(0, 0)]) and _valid(cfg, rec) == rm.rule(cfg, rec)


def test_the_bare_handle_refuses_some_pairs_and_a_geometry_record_fixes_them():
    cfg = _handle(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_POINT, True)
    refused = [t for t in rm.TYPES if not _valid(cfg, rm.record(*t))]
    assert (capi.ROBOT_UNICYCLE, capi.FOOTPRINT_POLYGON) in refused and (capi.ROBOT_SIMPLE_CAR, capi.FOOTPRINT_POINT) in refused
    assert (capi.ROBOT_UNICYCLE, capi.FOOTPRINT_POINT) not in refused
    rng = np.random.default_rng(5)
    for t in refused:
        assert _valid(cfg, rm.record(*t), _geometry_for(*t, rng))
    # a polygon record with a geometry record whose n_poly is not integral, or a vertex in use not finite
    g = _geometry_for(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_POLYGON, rng)
    g2 = g.copy(); g2[rg.NP] = 3.5
    g3 = g.copy(); g3[rg.XY + 1] = np.inf
    for bad in (g2, g3):
        assert not _valid(cfg, rm.record(0, 4), bad) and not rm.rule(cfg, rm.record(0, 4), bad)


def test_random_records_match_the_rule():
    rng = np.random.default_rng(11)
    pool = np.array([np.nan, np.inf, -np.inf, -1.0, -0.0, 0.0, 1.0, 2.0, 3.0, 4.0, 0.5, 5.0])
    for i in range(3000):
        t = rm.TYPES[int(rng.integers(20))]
        cfg = _handle(*t, bool(i % 2))
        rec = rng.choice(pool, 2)
        g = None if rng.random() < 0.4 else _geometry_for(*rm.TYPES[int(rng.integers(20))], rng, nan_unread=bool(rng.random() < 0.5))
        assert _valid(cfg, rec, g) == rm.rule(cfg, rec, g), f"{t} {rec} {g}"


@pytest.mark.parametrize("robot,footprint", rm.TYPES)
def test_patch_sets_exactly_the_two_types(robot, footprint):
    cfg = _handle(robot, footprint, False)
    for t in rm.TYPES:
        got = cfg.copy()
        _lib().emu_apply_robot_model(C.byref(got), _dp(rm.record(*t)))
        want = rm.with_model(cfg, rm.record(*t))
        assert C.string_at(C.addressof(got), C.sizeof(got)) == C.string_at(C.addressof(want), C.sizeof(want))
    got = cfg.copy()
    _lib().emu_apply_robot_model(C.byref(got), _dp(np.array([-0.0, -0.0])))
    assert (got.robot_type, got.footprint_type) == (0, 0)


def test_the_fleet_groups_are_valid_together():
    for host in (configs.cfg3(), configs.cfg2()):
        model, limits, geometry = rm.fleet_records(host, 8)
        for b in range(8):
            assert _valid(host, model[b], geometry[b]) and rm.rule(host, model[b], geometry[b])
            assert rg.rule(rm.group_config(host, rm.GROUPS[b % 4]), geometry[b])
        assert {tuple(m) for m in model} == {(0, 1), (1, 4), (2, 2), (3, 3)}


# ---- the per-robot-model solve kernels: -Xptxas -v lines and occupancy ----
_ENTRY = re.compile(r"Compiling entry function '(_Z\d+solve_fused(?:_models|_robot)?_kernel\w+)' for 'sm_90a'\n"
                    r"ptxas info\s+: Function properties for \1\n(.*)\n(ptxas info\s+: Used .*)")
_ANY_ENTRY = re.compile(r"Compiling entry function '(\w+)'")
_USED = re.compile(r"Used (\d+) registers, .* (\d+) bytes smem")
_MODELS = "solve_fused_models_kernel"


def _entries(text):
    """{kernel: (stack / spill line, registers / smem line)} of the solve kernels in -Xptxas -v output"""
    return {m.group(1): (m.group(2).strip(), m.group(3).strip()) for m in _ENTRY.finditer(text)}


def _robot_of(models_name):
    """the solve_fused_robot_kernel instantiation with the same template arguments as a per-robot-model entry (three parameters
    fewer)"""
    return models_name.replace("25solve_fused_models_kernel", "24solve_fused_robot_kernel").replace("9RobotArgsPKdS5_S5_", "9RobotArgs")


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_models_kernels_ptxas_lines_and_occupancy(tmp_path):
    """The translation unit of the per-robot-model entries (mpcb200_models.cu) compiles exactly the 16 MODEL_GENERIC
    solve_fused_models_kernel instantiations, every one with its -Xptxas -v lines as recorded in
    tests/golden/ptxas_solve_fused_models.txt and the registers and shared memory of the per-robot-limits entry of the same variant
    (tests/golden/ptxas_solve_fused_robot.txt, whose test holds those equal to the base solve_fused_kernel's) -- so CUDA fits as
    many of its CTAs on an SM as of the base kernel's, for every image size."""
    import __graft_entry__ as g
    cmd = [g._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
           "-o", str(tmp_path / "k.cubin"), os.path.join(_ROOT, "mpc_local_planner_b200", "csrc", "mpcb200_models.cu")]
    text = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    models = _entries(text)
    assert all(_MODELS in k for k in _ANY_ENTRY.findall(text)) and len(_ANY_ENTRY.findall(text)) == len(models)
    with open(os.path.join(_HERE, "golden", "ptxas_solve_fused_models.txt")) as f:
        recorded = _entries(f.read())
    assert len(recorded) == 16 and models == recorded
    assert all("ELi0ELb" in k for k in models)   # MODEL_GENERIC only
    with open(os.path.join(_HERE, "golden", "ptxas_solve_fused_robot.txt")) as f:
        robot = _entries(f.read())
    for k, (_, used) in models.items():
        assert _USED.search(used).group(1) == "255"
        assert _USED.search(used).groups() == _USED.search(robot[_robot_of(k)][1]).groups(), f"{k}: {used} vs {robot[_robot_of(k)][1]}"


# ---- the Python setters without a device ----
def test_model_symbols_are_exported():
    assert "mpcb200_set_robot_model" in capi.EXPORTS and "mpcb200_set_robot_model_async" in capi.EXPORTS
    lib = capi.load_library()
    lib.mpcb200_set_robot_model, lib.mpcb200_set_robot_model_async   # noqa: B018


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
    for bad in (np.zeros(rm.W), np.zeros((2, rm.W - 1)), np.zeros((2, rm.W + 1)), np.zeros((1, 2, rm.W))):
        with pytest.raises(ValueError):
            s.set_robot_model(bad)
    assert s.lib.calls == []
    s.set_robot_model(None)
    assert [c[0] for c in s.lib.calls] == ["mpcb200_set_robot_model"] and s.lib.calls[0][1][1] == 0
