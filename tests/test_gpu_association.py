"""The association over long obstacle lists (dev_associate_list: the caller's list wider than the 64 resident slots) on the GPU.

  * Stage by stage against the oracle on the crafted cases of tests/assoc_cases.py (exact ties within and across 32-wide
    chunks, thresholds, the heading line, forced inclusions beyond K, K = 0 / 1 / 5 / 16, list lengths around 32, 64 and 2048,
    circle / line / dynamic obstacles with a fixed and a free dt, every footprint): the resident slots, their list indices
    (OBSGIDX) and the dropped count equal tests/assoc_cases.resident_model of the oracle's selection, slot by slot.
  * The persistent solve kernel keeps the list indices in shared scratch and copies them out: same slots and indices as the
    phase kernel.
  * Re-association in outer iterations 2 to 5 on the device's own iterates.
  * Bit identity of every solve path that runs the long-list association: fused and phased, the queue, the costmap chain,
    the device-memory entry point, per-robot records equal to the configuration; and multistart's copy of the winner's list
    indices."""
import numpy as np
import pytest

import assoc_cases as ac
import costmap_cases as cm
import parity as par
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

GROUPS = ac.groups()


def _mapped(slots, gidx):
    slots = slots.astype(np.int64)
    return np.where(slots >= 0, gidx.astype(np.int64)[np.clip(slots, 0, None)], -1)


def _crafted_state(g, B):
    """a phase-API handle with the group uploaded and its poses (and SC_DT) written, no cold-start repair pending"""
    d = g.batch()
    s = capi.BatchSolver(g.cfg, B, device=0)
    s.upload(d["x0"], d["xf"], None, 0.0, d["obstacles"], None)
    s.run_phase(capi.PHASE_INIT)
    s.ws_write(capi.F_X, d["X"])
    SC = s.ws_read(capi.F_SCAL)
    SC[:, capi.SC_COLD] = 0.0
    SC[:, capi.SC_DT] = d["dt"]
    s.ws_write(capi.F_SCAL, SC)
    return s, d


def _read_assoc(s):
    return s.ws_read(capi.F_OBSIDX), s.ws_read(capi.F_OBSGIDX), s.ws_read(capi.F_SCAL)[:, capi.SC_OBST_DROPPED]


@pytest.mark.parametrize("g", GROUPS, ids=[g.name for g in GROUPS])
def test_long_list_association_matches_oracle_and_slot_model(cuda_lib, orc, g):
    B = len(g.cases)
    s, _ = _crafted_state(g, B)
    s.run_phase(capi.PHASE_ASSOCIATE)
    OBS, GIDX, DROP = _read_assoc(s)
    s.close()
    K = g.cfg.k_max_obstacles_per_stage
    for b, case in enumerate(g.cases):
        what = f"{g.name}/{case.name}"
        sel = ac.oracle_selection(orc, g.cfg, case)
        slots, gidx, dropped = ac.resident_model(sel)
        np.testing.assert_array_equal(GIDX[b].astype(np.int64), gidx, err_msg=f"{what}: resident list indices")
        assert DROP[b] == dropped, f"{what}: dropped {DROP[b]}, model {dropped}"
        if K == 0:
            continue
        np.testing.assert_array_equal(OBS[b].astype(np.int64), slots, err_msg=f"{what}: resident slots")
        if not dropped:
            np.testing.assert_array_equal(_mapped(OBS[b], GIDX[b]), sel, err_msg=f"{what}: selection")


@pytest.mark.parametrize("g", [g for g in GROUPS if g.cfg.k_max_obstacles_per_stage > 0], ids=lambda g: g.name)
def test_fused_kernel_scratch_list_indices_equal_phase_kernel(cuda_lib, g):
    """the persistent kernel's association (list indices in shared scratch, copied to OBSGIDX) from the same written poses:
    a warm solve of one iteration keeps stages 1..N-2 as written, and its one association is what OBSIDX holds afterwards"""
    B = len(g.cases)
    s, d = _crafted_state(g, B)
    s.run_phase(capi.PHASE_ASSOCIATE)
    want = _read_assoc(s)
    s.close()
    f, _ = _crafted_state(g, B)
    f.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_FUSED)
    f.solve_resident(cold=False)
    got = _read_assoc(f)
    f.close()
    for a, b, nm in zip(got, want, ("OBSIDX", "OBSGIDX", "dropped")):
        np.testing.assert_array_equal(a, b, err_msg=f"{g.name}: {nm}")


def _costmap_data(cid, B, seed, M=500, dups=12):
    """robots on random costmaps (up to 500 point obstacles each) plus duplicated entries: next to the original and at the end"""
    cfg = configs.cfg2() if cid == 2 else configs.cfg3()
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.01, seed)
    s = capi.BatchSolver(cfg, B, device=0)
    (count, typ, par_), found = s.costmap_obstacles(cost, origin, res, pose, 0.3, M)
    s.close()
    assert count.max() >= 100 and (found <= M).all() and (count > dups).all()
    rng = np.random.default_rng(seed)
    W = M + 2 * dups
    t2 = np.zeros((B, W), dtype=np.int32); p2 = np.zeros((B, W, capi.OBST_STRIDE)); c2 = np.zeros(B, dtype=np.int32)
    for b in range(B):
        lst = list(range(count[b]))
        for j in sorted(rng.choice(count[b], dups, replace=False), reverse=True):
            lst.insert(j + 1, j)
        lst += list(rng.choice(count[b], dups, replace=False))
        c2[b] = len(lst)
        t2[b, :len(lst)] = typ[b, lst]; p2[b, :len(lst)] = par_[b, lst]
    data = dict(x0=pose, xf=goal, u_prev=np.zeros((B, 2)), u_prev_dt=0.2, obstacles=(c2, t2, p2), viapoints=None)
    return cfg, data, (cost, origin, res, pose, goal)


def _outer_cfg():
    cfg = configs.cfg2()
    cfg.outer_iterations = 5
    return cfg


def test_reassociation_in_outer_iterations_matches_oracle(cuda_lib, orc):
    """the phase kernels' outer loop on a long list: after the cold association, four more rounds of a few iterations then
    a re-association; each selection equals orc_associate on the device's own poses at that point"""
    cfg, data, _ = _costmap_data(2, 8, 21)
    B = 8
    s = capi.BatchSolver(cfg, B, device=0)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.run_phase(capi.PHASE_INIT)
    compared = 0
    for oi in range(5):
        X = s.ws_read(capi.F_X)
        dt = s.ws_read(capi.F_SCAL)[:, capi.SC_DT]
        s.run_phase(capi.PHASE_ASSOCIATE)
        OBS, GIDX, DROP = _read_assoc(s)
        for b in range(B if oi > 0 else 0):   # (the cold association runs before the repair moves the poses: see test_gpu_variants)
            o = orc.instance_from_batch(cfg, data, b)
            o.init_cold()
            o.arr("X")[:] = X[b]
            o.arr("SCAL")[capi.SC_DT] = dt[b]
            o.associate()
            slots, gidx, dropped = ac.resident_model(o.arr("OBSIDX").astype(np.int64))
            what = f"outer iteration {oi + 1}, robot {b}"
            np.testing.assert_array_equal(OBS[b].astype(np.int64), slots, err_msg=what)
            np.testing.assert_array_equal(GIDX[b].astype(np.int64), gidx, err_msg=what)
            assert DROP[b] == dropped, what
            compared += 1
        for _ in range(6):
            s.run_phase(capi.PHASE_EVAL); s.run_phase(capi.PHASE_KKT); s.run_phase(capi.PHASE_LINESEARCH)
    s.close()
    assert compared == 4 * B


def _same(a, b, what):
    par.assert_same_solves([a], [b], what)


def _fields(out):
    return {f: np.array(out[f], copy=True) for f in par.SOLVE_FIELDS}


@pytest.mark.parametrize("cid", [2, 3])
def test_solve_paths_are_bit_identical_on_long_lists(cuda_lib, cid):
    """costmap lists with duplicated entries: every solve path that runs the long-list association gives the same bits"""
    B = 16
    cfg, data, scene = _costmap_data(cid, B, 30 + cid)
    x0, xf, up, ob = data["x0"], data["xf"], data["u_prev"], data["obstacles"]
    # fused and phased, cold then warm
    fused, _ = par.solve_twice(cfg, data, B, capi.SOLVE_FUSED)
    phased, _ = par.solve_twice(cfg, data, B, capi.SOLVE_PHASED)
    par.assert_same_solves(fused, phased, f"cfg{cid}: fused and phased")
    # five outer iterations, fused and phased
    if cid == 2:
        o5 = _outer_cfg()
        f5, _ = par.solve_twice(o5, data, B, capi.SOLVE_FUSED)
        p5, _ = par.solve_twice(o5, data, B, capi.SOLVE_PHASED)
        par.assert_same_solves(f5, p5, "five outer iterations: fused and phased")
    # the queue (no instance block, the list indices in shared scratch only) and the cold batch
    s = capi.BatchSolver(cfg, B, device=0)
    q = _fields(s.solve_stream(x0, xf, up, 0.2, ob, None))
    s.close()
    _same(q, fused[0], f"cfg{cid}: solve_stream and the cold batch")
    # per-robot records equal to the configuration
    s = capi.BatchSolver(cfg, B, device=0)
    rec = np.array(list(cfg.u_lb) + list(cfg.u_ub) + list(cfg.du_lb) + list(cfg.du_ub) + [cfg.min_obstacle_dist])
    s.set_robot_limits(np.tile(rec, (B, 1)))
    r = [_fields(s.step(x0, xf, up, 0.2, ob, None)) for _ in range(2)]
    s.close()
    par.assert_same_solves(r, fused, f"cfg{cid}: per-robot records equal to the configuration")
    # the costmap chain and extraction then step (the chain's own lists: no duplicates)
    cost, origin, res, pose, goal = scene
    s = capi.BatchSolver(cfg, B, device=0)
    chain = _fields(s.step_from_costmaps(pose, goal, cost, origin, res, 0.3, 500, u_prev=up, u_prev_dt=0.2))
    ext, _ = s.costmap_obstacles(cost, origin, res, pose, 0.3, 500)
    s.close()
    s = capi.BatchSolver(cfg, B, device=0)
    step = _fields(s.step(pose, goal, up, 0.2, ext, None))
    s.close()
    _same(chain, step, f"cfg{cid}: step_from_costmaps and extraction + step")
    # the device-memory entry point
    torch = pytest.importorskip("torch")
    st = torch.cuda.Stream()
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")   # noqa: E731
    s = capi.BatchSolver(cfg, B, device=0)
    s.set_stream(st.cuda_stream)
    outs = []
    with torch.cuda.stream(st):
        for _ in range(2):
            res_ = s.step_async(dev(x0), dev(xf), dev(up), 0.2, tuple(dev(a) for a in ob))
            torch.cuda.synchronize()
            outs.append({k: v.cpu().numpy() for k, v in res_.items()})
    s.close()
    par.assert_same_solves(outs, fused, f"cfg{cid}: step_async and step")


def test_multistart_copies_the_winners_list_indices(cuda_lib):
    """robot b's resident slots and list indices after step_multistart are those of its winning candidate's slot w B + b"""
    B, K = 24, 3
    cfg, data, _ = _costmap_data(2, B, 41)
    s = capi.BatchSolver(cfg, B * K, device=0)
    moved = 0
    for t in range(2):
        x0 = data["x0"] + 0.05 * t * (data["xf"] - data["x0"]) * np.array([1.0, 1.0, 0.0])
        r = s.step_multistart(x0, data["xf"], K, hysteresis=2.0, u_prev=data["u_prev"], u_prev_dt=0.2,
                              obstacles=data["obstacles"])
        OBS, GIDX = s.ws_read(capi.F_OBSIDX, B * K), s.ws_read(capi.F_OBSGIDX, B * K)
        for b in range(B):
            w = int(r["winner"][b])
            np.testing.assert_array_equal(GIDX[b], GIDX[w * B + b], err_msg=f"step {t} robot {b} winner {w}")
            np.testing.assert_array_equal(_mapped(OBS[b], GIDX[b]), _mapped(OBS[w * B + b], GIDX[w * B + b]))
            moved += w > 0
    s.close()
    assert moved > 0
