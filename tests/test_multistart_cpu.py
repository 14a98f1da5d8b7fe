"""Multistart solves without a GPU: the ranked cold initial guess of the oracle and of the emulator of the device headers, the
selection rule on synthetic candidate tables, and the register budget of the existing solve kernels."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import multistart_rule as rule
import parity as par
from mpc_local_planner_b200 import capi, configs

CASES = [("cfg2", configs.cfg2, 2), ("cfg3", configs.cfg3, 3), ("cfg4", configs.cfg4, 4)]
B = 12


@pytest.mark.parametrize("name,make,cid", CASES)
def test_oracle_rank0_is_cold_init(orc, name, make, cid):
    cfg = make()
    data = configs.generate(cid, B)
    for b in range(B):
        a = orc.instance_from_batch(cfg, data, b)
        a.init_cold()
        r = orc.instance_from_batch(cfg, data, b)
        rule.oracle_init_cold_rank(r, 0)
        assert np.array_equal(a.arr("X"), r.arr("X")) and np.array_equal(a.arr("U"), r.arr("U")), f"{name} b={b}"
        assert a.arr("SCAL")[capi.SC_DT] == r.arr("SCAL")[capi.SC_DT]


@pytest.mark.parametrize("name,make,cid", CASES)
def test_oracle_ranks_permute_the_lines(orc, name, make, cid):
    cfg = make()
    n, N = cfg.initial_guess_bumps, int(cfg.n)
    data = configs.generate(cid, B)
    for b in range(B):
        Xs = rule.straight(cfg, data, b, orc)
        scores, nv = rule.scores(cfg, data, b, orc, Xs)
        order = rule.ranking(scores)
        ms = []
        for r in range(2 * n + 1):
            o = orc.instance_from_batch(cfg, data, b)
            rule.oracle_init_cold_rank(o, r)
            ms.append(rule.line_of(o.arr("X"), Xs, nv, N))
            if cfg.robot_type != capi.ROBOT_UNICYCLE and ms[-1] != 0:   # car-like: headings follow the bumped path
                X = o.arr("X")
                k = N // 3
                assert X[2, k] == pytest.approx(math.atan2(X[1, k + 1] - X[1, k - 1], X[0, k + 1] - X[0, k - 1]), abs=1e-15)
        assert sorted(ms) == list(range(-n, n + 1)), f"{name} b={b}: ranks give lines {ms}"
        for r in rule.clear_ranks(scores, order):
            assert ms[r] == order[r] - n, f"{name} b={b} rank {r}: line {ms[r]}, expected {order[r] - n} (scores {scores})"


@pytest.mark.parametrize("name,make,cid", CASES)
def test_emulator_ranked_init_matches_oracle(orc, emu, name, make, cid):
    cfg = make()
    n = cfg.initial_guess_bumps
    data = configs.generate(cid, B)
    checked = 0
    for b in range(B):
        Xs = rule.straight(cfg, data, b, orc)
        scores, _ = rule.scores(cfg, data, b, orc, Xs)
        for r in rule.clear_ranks(scores, rule.ranking(scores)):
            o = orc.instance_from_batch(cfg, data, b)
            rule.oracle_init_cold_rank(o, r)
            e = emu.instance_from_batch(cfg, data, b)
            rule.emu_init_cold_rank(e, r)
            np.testing.assert_allclose(e.field(capi.F_X), o.arr("X"), rtol=0, atol=par.EMU["x"], err_msg=f"{name} b={b} rank {r}")
            np.testing.assert_array_equal(e.field(capi.F_U), o.arr("U"))
            checked += 1
        e0, e1 = emu.instance_from_batch(cfg, data, b), emu.instance_from_batch(cfg, data, b)
        e0.init(force_cold=True); rule.emu_init_cold_rank(e1, 0)
        assert np.array_equal(e0.W, e1.W)
    assert checked >= B * (2 * n + 1) // 2


# ---- the selection rule on synthetic candidate tables ----
CONV, MAXI, NUM, INV, MAXT, SKIP = (capi.STATUS_CONVERGED, capi.STATUS_MAX_ITER, capi.STATUS_NUMERICAL_ERROR,
                                    capi.STATUS_INVALID_INPUT, capi.STATUS_MAX_TIME, capi.STATUS_SKIPPED)


def test_rule_every_status_combination():
    statuses = (CONV, MAXI, NUM, INV, MAXT, SKIP, -1)
    obj = [3.0, 2.0, 1.0]
    inf = [0.5, 0.2, 0.1]
    for s0 in statuses:
        for s1 in statuses:
            for s2 in statuses:
                w = rule.winner([s0, s1, s2], obj, inf, 1.0)
                conv = [k for k, s in ((1, s1), (2, s2)) if s == CONV]
                stopped = lambda s: s in (MAXI, MAXT, -1)   # noqa: E731
                if conv:
                    assert w == (2 if 2 in conv else 1)   # the least objective (improves on the incumbent's at h = 1)
                elif s0 == CONV or stopped(s0):
                    assert w == 0
                elif stopped(s2):
                    assert w == 2   # the least infeasibility
                elif stopped(s1):
                    assert w == 1
                else:
                    assert w == 0


def test_rule_threshold_and_hysteresis():
    # obj(c*) exactly at obj(0) - (1 - h)|obj(0)|: the incumbent stays
    assert rule.winner([CONV, CONV], [10.0, 9.0], [0, 0], 0.9) == 0
    assert rule.winner([CONV, CONV], [10.0, np.nextafter(9.0, 0)], [0, 0], 0.9) == 1
    assert rule.winner([CONV, CONV], [10.0, 10.0], [0, 0], 1.0) == 0
    # h > 1: a challenger may win while worse, up to (h - 1)|obj(0)|
    assert rule.winner([CONV, CONV], [10.0, 10.5], [0, 0], 1.1) == 1
    # a tiny hysteresis: the incumbent stays unless the challenger is far better
    assert rule.winner([CONV, CONV], [10.0, 1e-3], [0, 0], 1e-300) == 0


def test_rule_negative_and_zero_objective():
    # obj(0) < 0 (the via-point orientation term): the threshold is obj(0) - (1 - h)|obj(0)|, below obj(0)
    assert rule.winner([CONV, CONV], [-2.0, -2.5], [0, 0], 0.9) == 1     # -2.5 < -2.2
    assert rule.winner([CONV, CONV], [-2.0, -2.1], [0, 0], 0.9) == 0
    assert rule.winner([CONV, CONV], [0.0, -1e-12], [0, 0], 0.5) == 1
    assert rule.winner([CONV, CONV], [0.0, 0.0], [0, 0], 0.5) == 0
    assert rule.winner([CONV, CONV], [0.0, 1e-12], [0, 0], 2.0) == 0


def test_rule_ties_and_skipped():
    assert rule.winner([NUM, CONV, CONV], [0, 5.0, 5.0], [0, 0, 0], 1.0) == 1      # equal objectives: the lower k
    assert rule.winner([NUM, MAXI, MAXT], [0, 0, 0], [0, 0.3, 0.3], 1.0) == 1      # equal infeasibilities: the lower k
    assert rule.winner([INV, SKIP, SKIP], [0, 0, 0], [0, 0, 0], 1.0) == 0
    assert rule.winner([NUM, SKIP, MAXI], [0, -9.0, 0], [0, 0, 0.4], 1.0) == 2     # a skipped challenger never wins
    assert rule.winner([CONV, SKIP, SKIP], [1.0, -5.0, -5.0], [0, 0, 0], 1.0) == 0


def test_rule_from_scal_table():
    Bn, K = 3, 2
    scal = np.zeros((Bn * K, capi.SCAL_WORDS))
    scal[:, capi.SC_STATUS] = [CONV, NUM, MAXI, CONV, CONV, SKIP]
    scal[:, capi.SC_OBJ] = [4.0, 1.0, 0.0, 3.0, 2.0, 0.0]
    assert rule.winners_from_scal(scal, Bn, K, 1.0).tolist() == [1, 1, 0]


# ---- register budget of the existing solve kernels ----
_PTXAS = re.compile(r"Compiling entry function '(_Z\d+solve_fused_kernel\w+)'.*?Used (\d+) registers", re.S)
_FRAME = re.compile(r"Function properties for (_Z\d+solve_fused_kernel\w+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")


def _fused_budget(text):
    """(registers, stack frame, spill stores, spill loads) per solve_fused_kernel instantiation of the other calls, by the name
    the instantiation had before the multistart flag (MULTI = false: its trailing template argument dropped)"""
    regs = {m.group(1): int(m.group(2)) for m in _PTXAS.finditer(text)}
    frames = {m.group(1): tuple(int(x) for x in m.group(2, 3, 4)) for m in _FRAME.finditer(text)}
    out = {}
    for k in regs:
        if "ELb1EEv" in k:   # a multistart instantiation
            continue
        out[k.replace("ELb0EEv", "EEv")] = (regs[k],) + frames[k]
    return out


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_fused_kernels_keep_their_register_budget(tmp_path):
    """Every solve_fused_kernel instantiation: registers, stack frame and spills as recorded before multistart (the solve kernel
    is bound by instruction fetch; tests/golden/ptxas_solve_fused.txt holds the -Xptxas -v lines of the kernels)"""
    import __graft_entry__ as g
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [g._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
           "-o", str(tmp_path / "k.cubin"), os.path.join(root, "mpc_local_planner_b200", "csrc", "mpcb200.cu")]
    now = _fused_budget(subprocess.run(cmd, capture_output=True, text=True, check=True).stderr)
    with open(os.path.join(root, "tests", "golden", "ptxas_solve_fused.txt")) as f:
        before = _fused_budget(f.read())
    assert len(before) == 14 and now == before
