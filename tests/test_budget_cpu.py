"""solver/ipopt/max_cpu_time (src/controller.cpp:395-397) without a GPU: the config field and its validation through the C ABI,
and the termination path of the shared device header on the CPU warp emulator -- a solve whose time budget runs out just before
the evaluation of iteration j holds bit for bit what a solve with max_iter = j holds; only the status differs (MAX_TIME)."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

from mpc_local_planner_b200 import capi, configs
from tests.conftest import ROOT


def test_header_declares_the_field_last_and_the_status():
    hdr = open(os.path.join(ROOT, "include", "mpcb200.h")).read()
    body = re.search(r"typedef struct mpcb200_config \{(.*?)\} mpcb200_config;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    decls = [d.strip() for d in body.split(";") if d.strip()]
    assert decls[-1] == "double max_cpu_time"
    assert re.search(r"#define MPCB200_STATUS_MAX_TIME 4\b", hdr) and capi.STATUS_MAX_TIME == 4
    assert re.search(r"#define MPCB200_VERSION 101\b", hdr)


def test_default_is_no_budget_and_the_last_field(cuda_lib):
    assert capi.Config._fields_[-1] == ("max_cpu_time", C.c_double)
    assert capi.Config.max_cpu_time.offset == C.sizeof(capi.Config) - 8
    assert capi.default_config().max_cpu_time == -1.0
    c = capi.Config()
    cuda_lib.mpcb200_default_config(C.byref(c))
    assert c.max_cpu_time == -1.0


def test_nan_budget_rejected(cuda_lib):
    h = C.c_void_p()
    c = capi.default_config(); c.max_cpu_time = math.nan
    assert cuda_lib.mpcb200_create(C.byref(c), 4, 0, C.byref(h)) == capi.E_INVALID
    assert b"max_cpu_time" in cuda_lib.mpcb200_last_error(None)
    # no budget (<= 0, +inf) and finite budgets pass the validation (without a device: E_NODEVICE)
    for t in (-1.0, 0.0, math.inf, 1e-9, 0.05, 1e6):
        c = capi.default_config(); c.max_cpu_time = t
        rc = cuda_lib.mpcb200_create(C.byref(c), 4, 0, C.byref(h))
        assert rc != capi.E_INVALID, t
        if rc == 0:
            cuda_lib.mpcb200_destroy(h)


def _midpoint():
    c = configs.cfg2(tol=1e-8)
    c.collocation = capi.COLLOC_MIDPOINT
    return c


# cfg 2: fixed dt; cfg 3: free dt (bordered KKT system); cfg 2 with midpoint differences: the LINES paths of the stage bodies
CASES = {"cfg2": (lambda: configs.cfg2(tol=1e-8), 2), "cfg3": (lambda: configs.cfg3(tol=1e-8), 3), "midpoint": (_midpoint, 2)}


@pytest.fixture(scope="module")
def budget_emu(emu, tmp_path_factory):
    """tests/emu/emu_budget.cpp (the emulator with a budget that runs out at a chosen iteration), built into a temporary directory"""
    src = os.path.join(ROOT, "tests", "emu", "emu_budget.cpp")
    lib = str(tmp_path_factory.mktemp("emu_budget") / "libemu_budget.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-march=x86-64-v3", "-fPIC", "-std=c++17", "-shared", "-o", lib, src, "-lm"])
    L = C.CDLL(lib)
    cp, dp = C.POINTER(capi.Config), C.POINTER(C.c_double)
    L.emu_init.argtypes = [cp, dp, C.c_int]
    L.emu_associate.argtypes = [cp, dp, C.c_double, C.c_int]
    L.emu_solve.argtypes = [cp, dp, C.c_double, C.c_int]
    L.emu_solve_expiring.argtypes = [cp, dp, C.c_double, C.c_int, C.c_int]
    L.emu_outputs.argtypes = [cp, dp, dp, dp]
    return L


class _Inst:
    """one instance block (inputs scattered by the emulator's binding) driven by the budget build of the emulator"""

    def __init__(self, L, emu, cfg, data, b):
        self.L, self.e = L, emu.instance_from_batch(cfg, data, b)
        self.cfg, self.W = self.e.cfg, self.e.W

    def _args(self):
        return C.byref(self.cfg), self.W.ctypes.data_as(C.POINTER(C.c_double))

    def solve(self):
        return self.L.emu_solve(*self._args(), self.e.u_prev_dt, 0)

    def solve_expiring(self, j):
        return self.L.emu_solve_expiring(*self._args(), self.e.u_prev_dt, 0, int(j))

    def guess(self):
        self.L.emu_init(*self._args(), 0)
        self.L.emu_associate(*self._args(), self.e.u_prev_dt, 1)

    def scal(self):
        return self.e.field(capi.F_SCAL)

    def outputs(self):
        N = self.e.N
        u, x = np.empty((N, 2)), np.empty((N, 3))
        self.L.emu_outputs(*self._args(), u.ctypes.data_as(C.POINTER(C.c_double)), x.ctypes.data_as(C.POINTER(C.c_double)))
        return u, x


def _state(e):
    """the whole instance block as bits, the status word masked"""
    w = e.W.copy().view(np.uint64)
    w[capi.SC_STATUS] = 0   # SCAL is the first field of the block
    return w


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("b", [0, 3])
def test_expiry_equals_max_iter(emu, budget_emu, case, b):
    make_cfg, cid = CASES[case]
    cfg = make_cfg()
    data = configs.generate(cid, b + 1)
    full = _Inst(budget_emu, emu, cfg, data, b)
    st_full = full.solve()
    n_it = int(full.scal()[capi.SC_ITER])
    assert n_it >= 4, (case, b, n_it)
    for j in sorted({0, 1, 2, n_it // 2, n_it - 1}):
        e = _Inst(budget_emu, emu, cfg, data, b)
        st = e.solve_expiring(j)
        capped = cfg.copy(); capped.max_iter = j
        r = _Inst(budget_emu, emu, capped, data, b)
        st_r = r.solve()
        assert st == capi.STATUS_MAX_TIME and st_r == capi.STATUS_MAX_ITER, (j, st, st_r)
        assert int(e.scal()[capi.SC_ITER]) == j
        np.testing.assert_array_equal(_state(e), _state(r))
        u, x = e.outputs(); ur, xr = r.outputs()
        np.testing.assert_array_equal(u, ur); np.testing.assert_array_equal(x, xr)
    # a budget that runs out after the natural end changes nothing, the status included
    for j in (n_it + 1, n_it + 10):
        e = _Inst(budget_emu, emu, cfg, data, b)
        assert e.solve_expiring(j) == st_full
        np.testing.assert_array_equal(e.W.view(np.uint64), full.W.view(np.uint64))


def test_expiry_at_the_start_is_the_initial_guess_and_ends_the_outer_iterations(emu, budget_emu):
    """expiry before the first evaluation: iters 0, the initial guess (init + association) as the result; with five outer
    iterations the solve stops after the first, as with one."""
    cfg = configs.cfg1(tol=1e-8); cfg.n = 30; cfg.k_max_obstacles_per_stage = 4
    data = configs.generate(2, 2)
    g = _Inst(budget_emu, emu, cfg, data, 1)
    g.guess()
    res = {}
    for outer in (1, 5):
        c = cfg.copy(); c.outer_iterations = outer
        e = _Inst(budget_emu, emu, c, data, 1)
        assert e.solve_expiring(0) == capi.STATUS_MAX_TIME
        assert e.scal()[capi.SC_ITER] == 0 and e.scal()[capi.SC_COLD] == 0
        np.testing.assert_array_equal(e.e.field(capi.F_X), g.e.field(capi.F_X))
        np.testing.assert_array_equal(e.e.field(capi.F_U), g.e.field(capi.F_U))
        res[outer] = e.W.copy()
    np.testing.assert_array_equal(res[1].view(np.uint64), res[5].view(np.uint64))
