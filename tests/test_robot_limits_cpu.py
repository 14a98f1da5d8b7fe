"""Per-robot limits without a GPU: the validity check and the configuration patch of the device headers (shared by the blocking
setter, the solve kernel and the emulator) against numpy restatements, and the compiled per-robot solve kernels against their
recorded -Xptxas -v lines and the occupancy of the kernels they are a form of."""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from mpc_local_planner_b200 import capi, configs

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB = []


def _lib():
    """the emulator with the two functions exported (tests/robot_limits/), compiled with the flags of emu/Makefile"""
    if not _LIB:
        out = os.path.join(tempfile.mkdtemp(prefix="mpcb200_robot_limits_"), "robot_limits_emu.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-march=x86-64-v3", "-fPIC", "-std=c++17", "-shared", "-o", out,
                               os.path.join(_HERE, "robot_limits", "robot_limits_emu.cpp"), "-lm"], stdout=subprocess.DEVNULL)
        lib = C.CDLL(out)
        lib.emu_robot_limits_valid.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_limits.argtypes = [C.POINTER(capi.Config), C.POINTER(C.c_double)]
        lib.emu_apply_robot_limits.restype = None
        _LIB.append(lib)
    return _LIB[0]


def _valid(cfg, rec):
    r = np.ascontiguousarray(rec, dtype=np.float64)
    return bool(_lib().emu_robot_limits_valid(C.byref(cfg), r.ctypes.data_as(C.POINTER(C.c_double))))


def _record(cfg):
    return np.array(list(cfg.u_lb) + list(cfg.u_ub) + list(cfg.du_lb) + list(cfg.du_ub) + [cfg.min_obstacle_dist])


def _rule(cfg, r):
    """the rules of mpcb200.h restated: no NaN, u_ub > u_lb, each bound finite exactly where the configuration's is, clearance in
    [0, inf)"""
    if np.isnan(r).any():
        return False
    cr = _record(cfg)
    lower = [0, 1, 4, 5]   # words holding lower bounds: finite means > -INF; the others are upper bounds: finite means < INF
    for w in range(8):
        on = (lambda v: v > -capi.INF) if w in lower else (lambda v: v < capi.INF)
        if on(r[w]) != on(cr[w]):
            return False
    return bool((r[2:4] > r[0:2]).all()) and 0.0 <= r[8] < np.inf


def _configs():
    c_on = configs.cfg2()                        # every control row on
    c_off = configs.cfg1()                       # control-rate rows off (+-INF)
    c_mixed = configs.cfg2()
    c_mixed.u_lb[1] = -capi.INF; c_mixed.du_ub[0] = capi.INF   # some rows off
    return [("all_on", c_on), ("rates_off", c_off), ("mixed", c_mixed)]


@pytest.mark.parametrize("name,cfg", _configs())
def test_validity_matches_the_rules(name, cfg):
    base = _record(cfg)
    specials = [np.nan, np.inf, -np.inf, capi.INF, -capi.INF, 0.0, -0.0]
    checked = 0
    for w, v in itertools.product(range(capi.LIMIT_WORDS), specials):   # one special value per word
        r = base.copy(); r[w] = v
        assert _valid(cfg, r) == _rule(cfg, r), f"{name}: word {w} = {v}"
        checked += 1
    for i in range(2):   # swapped, equal and nearly equal control bounds
        for lo, hi in ((0.3, -0.2), (0.1, 0.1), (0.1, np.nextafter(0.1, 1.0))):
            r = base.copy(); r[i], r[2 + i] = lo, hi
            assert _valid(cfg, r) == _rule(cfg, r), f"{name}: u bounds {i} = ({lo}, {hi})"
    for d in (-1e-300, -0.5, 0.0, 1e-300, 2.0, 1e300):   # clearance
        r = base.copy(); r[8] = d
        assert _valid(cfg, r) == _rule(cfg, r) == (d >= 0.0), f"{name}: clearance {d}"
    rng = np.random.default_rng(3)
    pool = np.array([np.nan, np.inf, -np.inf, capi.INF, -capi.INF, -1.0, -0.2, 0.0, 0.2, 1.0, 2e30])
    for _ in range(4000):   # random records: every word off, on, special or scaled, in every combination
        r = base * rng.uniform(0.5, 1.5, capi.LIMIT_WORDS)
        r = np.where(np.abs(base) >= capi.INF, base, r)
        hit = rng.random(capi.LIMIT_WORDS) < 0.2
        r[hit] = rng.choice(pool, hit.sum())
        assert _valid(cfg, r) == _rule(cfg, r), f"{name}: {r}"
        checked += 1
    assert _valid(cfg, base)
    assert checked > 4000


@pytest.mark.parametrize("cid", [2, 3, 4])
def test_patch_sets_exactly_the_nine_fields(cid):
    cfg = configs.config_for(cid)
    rng = np.random.default_rng(cid)
    for _ in range(20):
        rec = rng.uniform(-3.0, 3.0, capi.LIMIT_WORDS)
        got = cfg.copy()
        _lib().emu_apply_robot_limits(C.byref(got), np.ascontiguousarray(rec).ctypes.data_as(C.POINTER(C.c_double)))
        want = cfg.copy()
        want.u_lb[:] = rec[0:2]; want.u_ub[:] = rec[2:4]; want.du_lb[:] = rec[4:6]; want.du_ub[:] = rec[6:8]
        want.min_obstacle_dist = rec[8]
        assert C.string_at(C.addressof(got), C.sizeof(got)) == C.string_at(C.addressof(want), C.sizeof(want))


# ---- the per-robot solve kernels: -Xptxas -v lines and occupancy ----
_ENTRY = re.compile(r"Compiling entry function '(_Z\d+solve_fused(?:_robot)?_kernel\w+)' for 'sm_90a'\n"
                    r"ptxas info\s+: Function properties for \1\n(.*)\n(ptxas info\s+: Used .*)")
_USED = re.compile(r"Used (\d+) registers, .* (\d+) bytes smem")
_ROBOT = "solve_fused_robot_kernel"


def _entries(text):
    """{kernel: (stack / spill line, registers / smem line)} of the solve kernels in -Xptxas -v output"""
    return {m.group(1): (m.group(2).strip(), m.group(3).strip()) for m in _ENTRY.finditer(text)}


def _base_of(robot_name):
    """the solve_fused_kernel instantiation a per-robot entry is the form of (same template arguments, two parameters fewer)"""
    return robot_name.replace("24solve_fused_robot_kernel", "18solve_fused_kernel").replace("9FusedArgs9RobotArgs", "9FusedArgs")


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_robot_kernels_ptxas_lines_and_occupancy(tmp_path):
    """Every solve_fused_robot_kernel instantiation: its -Xptxas -v lines as recorded in tests/golden/ptxas_solve_fused_robot.txt,
    and the launch bound, registers and shared memory of its base kernel -- so CUDA fits as many of its CTAs on an SM as of the
    base kernel's, for every image size (the occupancy the host computes with cudaOccupancyMaxActiveBlocksPerMultiprocessor)."""
    import __graft_entry__ as g
    cmd = [g._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
           "-o", str(tmp_path / "k.cubin"), os.path.join(_ROOT, "mpc_local_planner_b200", "csrc", "mpcb200.cu")]
    now = _entries(subprocess.run(cmd, capture_output=True, text=True, check=True).stderr)
    robot = {k: v for k, v in now.items() if _ROBOT in k}
    with open(os.path.join(_HERE, "golden", "ptxas_solve_fused_robot.txt")) as f:
        recorded = _entries(f.read())
    assert len(recorded) == 28 and robot == recorded
    for k, (_, used) in robot.items():
        base = now[_base_of(k)][1]
        assert _USED.search(used).groups() == _USED.search(base).groups(), f"{k}: {used} vs {base}"
