"""mpcb200_step_batch_multistart on the GPU: K = 1 is mpcb200_step_batch, the winners follow the selection rule from the candidates'
SCAL words, a winning challenger's state moves into the robot's slot, challengers are the oracle's cold solves from their rank,
execution options do not change results, arguments are validated, and the C++ mirror binds it."""
import numpy as np
import pytest

import multistart_rule as rule
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

CFGS = {2: configs.cfg2, 3: configs.cfg3, 4: configs.cfg4}
OUT = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")
STATE = (capi.F_X, capi.F_U, capi.F_NU, capi.F_S, capi.F_LAM, capi.F_OBSIDX, capi.F_SCAL)
WARM = STATE   # what a warm start reads of a slot


def _same(a, b, what):
    for k in OUT:
        assert np.array_equal(a[k], b[k]), f"{what}: {k} differs"


def _moved(data, t):
    """the robots a little further along: start poses shifted towards the goal (a warm step's measurement)"""
    d = dict(data)
    d["x0"] = data["x0"] + t * (data["xf"] - data["x0"]) * np.array([1.0, 1.0, 0.0])
    return d


def _step(s, d, **kw):
    return s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"], **kw)


def _ms(s, d, K, **kw):
    return s.step_multistart(d["x0"], d["xf"], K, u_prev=d["u_prev"], u_prev_dt=d["u_prev_dt"], obstacles=d["obstacles"],
                             viapoints=d["viapoints"], **kw)


@pytest.mark.parametrize("cid", [2, 3, 4])
def test_k1_is_step_batch(cid):
    cfg, B = CFGS[cid](), 24
    data = configs.generate(cid, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    for t in range(4):
        d = _moved(data, 0.05 * t)
        ra, rb = _ms(a, d, 1), _step(b, d)
        _same(ra, rb, f"cfg{cid} step {t}")
        assert (ra["winner"] == 0).all()
    a.close(); b.close()


@pytest.mark.parametrize("cid", [2, 3])
def test_winners_follow_the_rule_and_move_their_state(cid):
    """the incumbent's SCAL words come from a twin handle that runs mpcb200_step_batch from the same state (a winning challenger
    overwrites slot b), the challengers' from their slots"""
    cfg, B, K = CFGS[cid](), 32, 3
    data = configs.generate(cid, B)
    s, twin = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B)
    for t in range(2):
        d = _moved(data, 0.05 * t)
        if t:
            for f in WARM:
                twin.ws_write(f, s.ws_read(f, B))
        inc = _step(twin, d)
        r = _ms(s, d, K)
        scal = s.ws_read(capi.F_SCAL, B * K)
        table = scal.copy()
        table[:B] = twin.ws_read(capi.F_SCAL, B)
        assert np.array_equal(rule.winners_from_scal(table, B, K, 1.0), r["winner"]), f"step {t}"
        assert (r["winner"] > 0).any()
        keep = r["winner"] == 0
        for k in OUT:
            assert np.array_equal(r[k][keep], inc[k][keep]), k
        for f in STATE:
            a = s.ws_read(f, B * K)
            for b in np.nonzero(r["winner"])[0]:
                w = int(r["winner"][b])
                assert np.array_equal(a[b], a[w * B + b]), f"field {f} robot {b}"
        X, U = s.ws_read(capi.F_X, B), s.ws_read(capi.F_U, B)
        assert np.array_equal(r["x_seq"][:, :, :2], X.transpose(0, 2, 1)[:, :, :2])
        assert np.array_equal(r["u_seq"][:, :-1], U.transpose(0, 2, 1)[:, :-1])
        assert np.array_equal(r["dt"], scal[:B, capi.SC_DT])
    s.close(); twin.close()


@pytest.mark.parametrize("cid", [2, 3])
def test_challengers_are_oracle_cold_solves_at_their_rank(orc, cid):
    cfg, B, K = CFGS[cid](tol=1e-8), 8, 3
    data = configs.generate(cid, B)
    s = capi.BatchSolver(cfg, B * K)
    _ms(s, data, K)
    st = s.ws_read(capi.F_SCAL, B * K)[:, capi.SC_STATUS]
    U = s.ws_read(capi.F_U, B * K)
    compared = 0
    for b in range(B):
        clear = rule.clear_ranks(rule.scores(cfg, data, b, orc, rule.straight(cfg, data, b, orc))[0], list(range(2 * cfg.initial_guess_bumps + 1)))
        for k in range(1, K):
            if k not in clear:   # a near-tie of the ranking: the device may take the other line
                continue
            o = orc.instance_from_batch(cfg, data, b)
            rule.oracle_init_cold_rank(o, k)
            u, x, res = orc.instance_from_batch(cfg, data, b).step(x_init=o.arr("X").T.copy())   # the cold solve from that line
            assert res.status == int(st[k * B + b]), f"cfg{cid} robot {b} challenger {k}"
            if res.status == capi.STATUS_CONVERGED:
                du = np.abs(U[k * B + b].T[:-1] - u[:-1]).max()
                assert du < 1e-4, f"cfg{cid} robot {b} challenger {k}: |du| = {du}"
                compared += 1
    assert compared >= B * (K - 1) // 2
    s.close()


def test_tiny_hysteresis_keeps_converged_incumbents():
    cfg, B, K = configs.cfg2(), 64, 3
    data = configs.generate(2, B)
    a, b = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B)
    ra, rb = _ms(a, data, K, hysteresis=1e-300), _step(b, data)
    conv = rb["status"] == capi.STATUS_CONVERGED
    assert conv.sum() > B // 2
    for k in OUT:
        assert np.array_equal(ra[k][conv], rb[k][conv]), k
    assert (ra["winner"][conv] == 0).all()
    a.close(); b.close()


def test_next_step_warm_starts_from_the_winner():
    cfg, B, K = configs.cfg2(), 48, 3
    data = configs.generate(2, B)
    a, b = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B)
    _ms(a, data, K)
    _step(b, data)   # fills the slots' layout; every field of slot b is then overwritten with the multistart's
    for f in WARM:
        b.ws_write(f, a.ws_read(f, B))
    d = _moved(data, 0.05)
    _same(_step(a, d), _step(b, d), "step after multistart")
    a.close(); b.close()


def test_execution_options_do_not_change_results():
    cfg, B, K = configs.cfg2(), 400, 3
    data = configs.generate(2, B)
    ref = None
    for opt, val in ((capi.OPT_ORDER_BY_HISTORY, 0), (capi.OPT_ORDER_BY_HISTORY, 1), (capi.OPT_CTAS_PER_SM, 1), (capi.OPT_CTAS_PER_SM, 2)):
        s = capi.BatchSolver(cfg, B * K)
        s.set_option(opt, val)
        outs = [_ms(s, _moved(data, 0.05 * t), K) for t in range(2)]   # the second call is ordered by the first's history
        if ref is None:
            ref = outs
        for o, r in zip(outs, ref):
            _same(o, r, f"option {opt}={val}")
            assert np.array_equal(o["winner"], r["winner"])
        s.close()


def test_time_budget_statuses_follow_rule_2():
    """candidates stopped by max_cpu_time: with none converged the incumbent stays when it was stopped, else the stopped challenger
    with the least infeasibility wins (a winning challenger overwrites the incumbent's slot: there only the challengers' part of the
    rule is checked)"""
    cfg, B, K = configs.cfg2(), 256, 3
    cfg.max_cpu_time = 2e-4
    data = configs.generate(2, B)
    s = capi.BatchSolver(cfg, B * K)
    r = _ms(s, data, K)
    scal = s.ws_read(capi.F_SCAL, B * K)
    st = scal[:, capi.SC_STATUS]
    assert (st == capi.STATUS_MAX_TIME).any()
    rule_w = rule.winners_from_scal(scal, B, K, 1.0)
    for b in range(B):
        w = int(r["winner"][b])
        if w == 0:
            assert rule_w[b] == 0, f"robot {b}"
            continue
        rows = scal[[k * B + b for k in range(K)]]
        assert np.array_equal(rows[0], rows[w])
        ch = rows.copy()
        ch[0, capi.SC_STATUS] = capi.STATUS_NUMERICAL_ERROR   # the incumbent lost: neither converged nor stopped, or worse
        if (rows[1:, capi.SC_STATUS] == capi.STATUS_CONVERGED).any():
            ch[0, capi.SC_STATUS] = capi.STATUS_MAX_ITER
        assert rule.winner(ch[:, capi.SC_STATUS], ch[:, capi.SC_OBJ], ch[:, capi.SC_INF], 1.0) == w, f"robot {b}"
    s.close()


def test_validation():
    cfg, B = configs.cfg2(), 16
    data = configs.generate(2, B)
    s = capi.BatchSolver(cfg, 10 * B)
    bad = [dict(K=0), dict(K=11), dict(K=2 * cfg.initial_guess_bumps + 2), dict(K=2, hysteresis=0.0), dict(K=2, hysteresis=-1.0),
           dict(K=2, hysteresis=float("nan")), dict(K=2, hysteresis=float("inf"))]
    for kw in bad:
        K = kw.pop("K")
        with pytest.raises(capi.SolverError, match=r"\(-1\)"):
            _ms(s, data, K, **kw)
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_PHASED)
    with pytest.raises(capi.SolverError, match=r"\(-2\)"):
        _ms(s, data, 2)
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_FUSED)
    c2 = configs.cfg2(); c2.reference_initial_guess = 1
    r = capi.BatchSolver(c2, 2 * B)
    with pytest.raises(capi.SolverError, match=r"\(-2\)"):
        _ms(r, data, 2)
    r.close()
    fresh = capi.BatchSolver(cfg, 10 * B)
    _same(_step(s, data), _step(fresh, data), "after the refused calls")
    s.close(); fresh.close()


def test_property_b1024():
    cfg, B, K = configs.cfg2(), 1024, 3
    data = configs.generate(2, B)
    s, twin = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B)
    r, t = _ms(s, data, K), _step(twin, data)
    scal = s.ws_read(capi.F_SCAL, B * K)
    st = scal[:, capi.SC_STATUS].reshape(K, B)
    some = (st == capi.STATUS_CONVERGED).any(axis=0)
    assert np.array_equal(r["status"] == capi.STATUS_CONVERGED, some)
    inc = t["status"] == capi.STATUS_CONVERGED
    tw = twin.ws_read(capi.F_SCAL, B)[:, capi.SC_OBJ]
    won = scal[:B, capi.SC_OBJ]
    assert (won[inc] <= tw[inc]).all()
    s.close(); twin.close()


def test_cpp_mirror_multistart_matches_python():
    """the demo scenario through the C++ Controller with multistart_candidates = 3: every step converges, and the first step
    equals BatchSolver.step_multistart at B = 1"""
    import os
    import re
    import subprocess
    from tests.conftest import ROOT
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples"), "-B", "test_mpc_optim_demo"], stdout=subprocess.DEVNULL)
    p = subprocess.run([os.path.join(ROOT, "examples", "test_mpc_optim_demo"), "3", "0", "-1", "3"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr
    rows = re.findall(r"step (\d+) ok 1 status (\d+) iters (\d+) dt (\S+) u0 (\S+) (\S+)", p.stdout)
    assert len(rows) == 3 and all(r[1] == "0" for r in rows), p.stdout
    cfg = capi.default_config()
    cfg.k_max_obstacles_per_stage = 3
    cfg.tol = 1e-8
    count = np.array([3], dtype=np.int32)
    types = np.full((1, 3), capi.OBST_POINT, dtype=np.int32)
    params = np.zeros((1, 3, capi.OBST_STRIDE))
    params[0, :, :2] = [[-3, 1], [6, 2], [4, 0.1]]
    s = capi.BatchSolver(cfg, 3)
    r = s.step_multistart(np.zeros((1, 3)), np.array([[5.0, 2.0, 0.0]]), 3, obstacles=(count, types, params), reinit=np.ones(1))
    assert int(rows[0][2]) == r["iters"][0]
    assert float(rows[0][3]) == pytest.approx(r["dt"][0], abs=1e-9)
    assert float(rows[0][4]) == pytest.approx(r["u_seq"][0, 0, 0], abs=1e-9)
    assert float(rows[0][5]) == pytest.approx(r["u_seq"][0, 0, 1], abs=1e-9)
    s.close()
