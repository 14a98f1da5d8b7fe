"""Crafted obstacle-association cases and the resident-slot model of the association over long lists -- TEST INFRASTRUCTURE.

Every case fixes the pose of each stage (X is written directly, not produced by a cold start) and an obstacle list.  Where the
outcome turns on an exact comparison (equal distances, a distance equal to force_inclusion_dist or cutoff_dist, a centroid on
the heading line) the poses have heading 0 and every coordinate is a multiple of 1/8 m: the distances are then exact in any
evaluation order, with or without fused multiply-adds, so both sides of a comparison see the same numbers.

A case group shares one configuration (one handle on the device); the cases of a group are the rows of one batch, their lists
padded to the group's array width.  The width is always larger than the 64 resident slots, so the device associates over the
list in global memory (dev_associate_list) even where the count is small.

The association rule (stage_inequality_se2.cpp:73-147 with the project's K row slots): forced inclusions (dist <
force_inclusion_dist, and every dynamic obstacle) in list order, then the nearest left and the nearest right obstacle within
cutoff_dist, the earliest on equal distances; each goes into the K slots -- appended while there is room, otherwise it replaces
the FIRST farthest slot if it is nearer.  `restated_selection` applies that slot rule to the numpy restatement of the reference
(tests/golden/ocp_numpy.py).  `resident_model` allocates the resident slots as the long-list association documents it."""
import os
import sys

import numpy as np

from mpc_local_planner_b200 import capi, configs

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import ocp_numpy as on  # noqa: E402

M_RES = 64          # resident obstacle slots per instance (MAX_OBST)
LIST_MAX = 2048     # longest caller list (MAX_OBST_LIST)
FAR = -1.0e3        # filler obstacles sit beyond every cut-off
EIGHTH = 0.125


class Case:
    """one instance: X [N, 3] (stages 1..N-2 are associated), the obstacle list (types [n], params [n, 7]), SC_DT and tags
    naming the edges it is built to reach"""

    def __init__(self, name, X, types, params, dt, tags=()):
        self.name, self.X, self.dt, self.tags = name, np.asarray(X, dtype=np.float64), float(dt), tuple(tags)
        self.types = np.asarray(types, dtype=np.int32)
        self.params = np.asarray(params, dtype=np.float64).reshape(-1, capi.OBST_STRIDE)

    @property
    def count(self):
        return len(self.types)


class Group:
    def __init__(self, name, cfg, cases):
        self.name, self.cfg, self.cases = name, cfg, cases

    def width(self):
        return max(M_RES + 1, max(c.count for c in self.cases))

    def batch(self):
        """device inputs of the group: x0, xf, X [B, 3, N], obstacles (count, types, params) padded to width(), dt [B]"""
        B, W, N = len(self.cases), self.width(), int(self.cfg.n)
        count = np.array([c.count for c in self.cases], dtype=np.int32)
        types = np.zeros((B, W), dtype=np.int32)
        params = np.zeros((B, W, capi.OBST_STRIDE))
        params[:, :, 0] = FAR; params[:, :, 1] = FAR   # padding: never read, finite anyway
        X = np.zeros((B, 3, N))
        for b, c in enumerate(self.cases):
            types[b, :c.count] = c.types; params[b, :c.count] = c.params
            X[b] = c.X.T
        x0 = X[:, :, 0].copy(); xf = X[:, :, N - 1].copy()
        return dict(x0=x0, xf=xf, X=X, obstacles=(count, types, params), dt=np.array([c.dt for c in self.cases]))


# ---- the rule, restated ----
def is_dynamic(cfg, op):
    return bool(cfg.enable_dynamic_obstacles) and (op[5] != 0.0 or op[6] != 0.0)


def restated_selection(cfg, X, types, params, dt):
    """[K, N] list indices (-1: empty slot): ocp_numpy.associate's choice per stage, put into the K row slots in the project's
    order (forced and dynamic obstacles in list order, then left, then right) with the first-farthest replacement rule"""
    N, K = X.shape[0], int(cfg.k_max_obstacles_per_stage)
    out = -np.ones((max(K, 1), N), dtype=np.int64)
    if K == 0:
        return out
    keep = on.associate(cfg, X, types, params, dt)
    for k in range(1, N - 1):
        dist = {j: on.footprint_distance(cfg, X[k], types[j], params[j], t=k * dt) for j in keep[k]}
        forced = sorted(j for j in keep[k] if is_dynamic(cfg, params[j]) or dist[j] < cfg.force_inclusion_dist)
        sides = [j for j in keep[k] if j not in forced]   # left, then right (ocp_numpy's order)
        idx, dst = [], []
        for j in forced + sides:
            if len(idx) < K:
                idx.append(j); dst.append(dist[j])
                continue
            far = int(np.argmax(dst))   # the first farthest
            if dist[j] < dst[far]:
                idx[far], dst[far] = j, dist[j]
        out[:len(idx), k] = idx
    return out


def resident_model(sel, M=M_RES):
    """Resident slots of a long-list association from the full selection sel [K, N] (list indices, -1 empty): stages 1..N-2,
    then slot order within a stage; a list index not yet resident takes the next free slot; once M are taken, a new one is
    dropped (its row slot stays -1) and counted.  Returns (slots [K, N], gidx [M] (-1 beyond the last used), dropped)."""
    K, N = sel.shape
    slots = -np.ones_like(sel)
    gidx = -np.ones(M, dtype=np.int64)
    where, nres, dropped = {}, 0, 0
    for k in range(1, N - 1):
        for s in range(K):
            g = int(sel[s, k])
            if g < 0:
                continue
            if g not in where:
                if nres == M:
                    dropped += 1
                    continue
                where[g] = nres; gidx[nres] = g; nres += 1
            slots[s, k] = where[g]
    return slots, gidx, dropped


# ---- the oracle and the emulator on one case ----
def oracle_selection(orc, cfg, case):
    o = orc.Instance(cfg, case.X[0], case.X[-1], obst_types=case.types, obst_params=case.params)
    o.init_cold()
    o.arr("X")[:] = case.X.T
    o.arr("SCAL")[capi.SC_DT] = case.dt
    o.associate()
    return o.arr("OBSIDX").astype(np.int64).copy()


def emulator_selection(emu, cfg, case):
    """the short-list association (associate_stage) of the CPU warp emulator; lists of at most M_RES obstacles"""
    e = emu.EmuInstance(cfg, case.X[0], case.X[-1], obst_types=case.types, obst_params=case.params)
    e.set_field(capi.F_X, case.X.T)
    sc = e.field(capi.F_SCAL).copy()
    sc[capi.SC_COLD] = 0.0; sc[capi.SC_DT] = case.dt
    e.set_field(capi.F_SCAL, sc)
    e.associate(first_outer=False)
    return e.field(capi.F_OBSIDX).astype(np.int64)


# ---- case construction ----
def _stage_poses(N, spacing=20.0):
    """stage k at (spacing k, 0), heading 0: every stage sees only its own obstacles"""
    X = np.zeros((N, 3))
    X[:, 0] = spacing * np.arange(N)
    return X


class _List:
    """an obstacle list of n entries, fillers beyond every cut-off unless set"""

    def __init__(self, n):
        self.types = np.zeros(n, dtype=np.int32)
        self.params = np.zeros((n, capi.OBST_STRIDE))
        self.params[:, 0] = FAR - np.arange(n)   # distinct fillers
        self.params[:, 1] = FAR

    def point(self, j, x, y, v=(0.0, 0.0)):
        self.types[j] = capi.OBST_POINT
        self.params[j] = [x, y, 0.0, 0.0, 0.0, v[0], v[1]]

    def circle(self, j, x, y, r, v=(0.0, 0.0)):
        self.types[j] = capi.OBST_CIRCLE
        self.params[j] = [x, y, 0.0, 0.0, r, v[0], v[1]]

    def line(self, j, a, b, v=(0.0, 0.0)):
        self.types[j] = capi.OBST_LINE
        self.params[j] = [a[0], a[1], b[0], b[1], 0.0, v[0], v[1]]


def base_cfg(n=10, k=5):
    """cfg 2 (unicycle, point footprint, force_inclusion_dist 0.5, cutoff_dist 2.5) with a short horizon and K row slots"""
    cfg = configs.cfg2(n=n, tol=1e-6)
    cfg.k_max_obstacles_per_stage = k
    cfg.max_iter = 1
    cfg.warm_start = 0      # a warm solve keeps the written poses (no shift)
    return cfg


def ties_and_boundaries(N=10):
    """One stage per edge (K = 5, list of 2048):
      1  duplicates at (10, 11) on the left and a right obstacle at the same distance (12)
      2  duplicates at (31, 32) (the last lane of one chunk, the first of the next) and at (63, 64)
      3  duplicates at (5, 37) (one lane, two chunks) and at (96, 1000)
      4  duplicates at (0, 2047) (the first and the last entry) and at (100, 2000)
      5  mirrored pairs at equal distance on one side: (200, 300) on the left, (400, 401) on the right
      6  forced inclusions beyond K with equal distances: the replacement takes the first farthest slot
      7  dist == force_inclusion_dist (not forced: the left candidate), dist == cutoff_dist (kept: the right candidate),
         dist just above the cut-off (dropped), dist just below force_inclusion_dist (forced)
      8  a centroid on the heading line (cross product 0: the right side) nearer than the right and the left obstacle"""
    X = _stage_poses(N)
    L = _List(LIST_MAX)
    x = X[:, 0]
    L.point(10, x[1], 1.0); L.point(11, x[1], 1.0); L.point(12, x[1], -1.0); L.point(13, x[1], -1.0)
    L.point(31, x[2], 1.5); L.point(32, x[2], 1.5); L.point(63, x[2], -0.75); L.point(64, x[2], -0.75)
    L.point(5, x[3], 0.625); L.point(37, x[3], 0.625); L.point(96, x[3], -1.0); L.point(1000, x[3], -1.0)
    L.point(0, x[4], 1.25); L.point(2047, x[4], 1.25); L.point(100, x[4], -2.0); L.point(2000, x[4], -2.0)
    L.point(300, x[5] + 0.75, 1.0); L.point(200, x[5] - 0.75, 1.0)       # both at 1.25 on the left
    L.point(401, x[5] - 0.375, -0.5); L.point(400, x[5] + 0.375, -0.5)   # both at 0.625 on the right
    # stage 6: forced at 0.25, 0.375, 0.375, 0.125, 0.375 (K full), 0.25 (replaces the first 0.375), 0.375 (no), 0.125 (replaces
    # the next first 0.375); spread within and across chunks
    for j, (dx, dy) in zip([500, 501, 540, 541, 600, 700, 701, 900],
                           [(0.25, 0), (0, 0.375), (0, -0.375), (0.125, 0), (-0.375, 0), (-0.25, 0), (0.375, 0), (-0.125, 0)]):
        L.point(j, x[6] + dx, dy)
    L.point(950, x[6], 1.0)   # a left candidate, farther than every forced one: it replaces nothing
    # stage 7: the thresholds
    L.point(1100, x[7], 0.5)                                  # dist 0.5 == force_inclusion_dist: left candidate
    L.point(1101, x[7], -2.5)                                 # dist 2.5 == cutoff_dist: right candidate
    L.point(1102, x[7], -(2.5 + 1.0 / 1024))                  # just beyond the cut-off
    L.point(1103, x[7] - (0.5 - 1.0 / 1024), 0.0)             # just inside force_inclusion_dist: forced
    # stage 8: the heading line
    L.point(1200, x[8] + 1.0, 0.0)                            # centroid on the heading line, dist 1: right
    L.point(1201, x[8], 1.5)                                  # left, dist 1.5
    L.point(1202, x[8], -1.25)                                # right, dist 1.25
    return Case("ties_and_boundaries", X, L.types, L.params, 0.3,
                ("tie_in_chunk", "tie_across_chunks", "tie_same_lane", "tie_first_last", "tie_mirrored", "tie_forced",
                 "force_boundary", "cutoff_boundary", "heading_line"))


def _dense_points(rng, X, n, spread=3.0, dup_every=0):
    """n point obstacles on the 1/8 m grid around the stage poses (duplicates of earlier entries every dup_every entries)"""
    L = _List(n)
    lo, hi = X[1:-1, 0].min() - spread, X[1:-1, 0].max() + spread
    for j in range(n):
        if dup_every and j % dup_every == dup_every - 1:
            src = int(rng.integers(0, j))
            L.types[j], L.params[j] = L.types[src], L.params[src]
            continue
        L.point(j, np.round(rng.uniform(lo, hi) * 8) / 8, np.round(rng.uniform(-spread, spread) * 8) / 8)
    return L


def _dyadic_line_poses(rng, N, step=0.5):
    X = np.zeros((N, 3))
    X[:, 0] = step * np.arange(N)
    X[:, 1] = np.round(rng.uniform(-0.5, 0.5, N) * 8) / 8
    return X


def list_shapes(N=10):
    """counts 0, 1, 31, 32, 33, 63, 64, 65, 2047, 2048 of grid points around dyadic poses (heading 0), every 7th entry a
    duplicate of an earlier one: equal distances within a chunk and across chunks"""
    out = []
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 2047, 2048):
        rng = np.random.default_rng(1000 + n)
        X = _dyadic_line_poses(rng, N)
        L = _dense_points(rng, X, n, dup_every=7)
        out.append(Case(f"count_{n}", X, L.types, L.params, 0.3, ("list_shape",)))
    return out


def forced_cluster(N, k_slots, per_stage, seed):
    """per_stage point obstacles inside force_inclusion_dist of every stage (on the 1/8 m grid: many equal distances), then
    grid points around: more forced inclusions than the K slots"""
    rng = np.random.default_rng(seed)
    X = _stage_poses(N, spacing=10.0)
    n = per_stage * (N - 2) + 200
    L = _List(n)
    offs = [(dx / 8, dy / 8) for dx in range(-3, 4) for dy in range(-3, 4) if dx * dx + dy * dy < 16]
    j = 0
    order = rng.permutation(n - 200)   # the stages' clusters interleaved over the list
    for k in range(1, N - 1):
        pick = rng.choice(len(offs), per_stage, replace=True)
        for p in pick:
            L.point(int(order[j]), X[k, 0] + offs[p][0], offs[p][1]); j += 1
    for i in range(n - 200, n):
        k = int(rng.integers(1, N - 1))
        L.point(i, X[k, 0] + np.round(rng.uniform(-2.5, 2.5) * 8) / 8, np.round(rng.uniform(-2.5, 2.5) * 8) / 8)
    tags = ("forced_beyond_K",) + (("overflow",) if k_slots * (N - 2) > M_RES else ())   # K = 16: 128 rows over 8 stages
    return Case(f"forced_K{k_slots}", X, L.types, L.params, 0.3, tags)


def random_poses(N=10, seeds=(1, 2, 3)):
    """random headings and positions, random continuous obstacle positions (general coverage)"""
    out = []
    for s in seeds:
        rng = np.random.default_rng(2000 + s)
        X = np.zeros((N, 3))
        X[:, 0] = np.cumsum(rng.uniform(0.2, 0.6, N)); X[:, 1] = rng.normal(0, 0.3, N); X[:, 2] = rng.uniform(-np.pi, np.pi, N)
        n = int(rng.integers(70, 400))
        L = _List(n)
        for j in range(n):
            L.point(j, rng.uniform(-2, X[-1, 0] + 2), rng.uniform(-3, 3))
        out.append(Case(f"random_{s}", X, L.types, L.params, 0.3, ("random",)))
    return out


def typed_lists(N=10, seed=7):
    """points, circles (dyadic radii) and line segments in one long list, duplicates of circles and lines included"""
    rng = np.random.default_rng(seed)
    X = _dyadic_line_poses(rng, N)
    n = 300
    L = _List(n)
    lo, hi = X[1, 0] - 3, X[-2, 0] + 3
    for j in range(n):
        if j % 11 == 10:
            src = int(rng.integers(0, j)); L.types[j], L.params[j] = L.types[src], L.params[src]
            continue
        cx, cy = np.round(rng.uniform(lo, hi) * 8) / 8, np.round(rng.uniform(-3, 3) * 8) / 8
        kind = j % 3
        if kind == 0:
            L.point(j, cx, cy)
        elif kind == 1:
            L.circle(j, cx, cy, EIGHTH * int(rng.integers(1, 4)))
        else:
            ang = rng.uniform(0, np.pi)
            h = rng.uniform(0.2, 0.8)
            L.line(j, (cx - h * np.cos(ang), cy - h * np.sin(ang)), (cx + h * np.cos(ang), cy + h * np.sin(ang)))
    return Case("typed", X, L.types, L.params, 0.3, ("circle", "line"))


def dynamic_list(N, dt, seed):
    """static grid points and a dozen moving obstacles (more than K: forced at every stage, the slots by distance at t = k dt)"""
    rng = np.random.default_rng(seed)
    X = _dyadic_line_poses(rng, N)
    n = 150
    L = _dense_points(rng, X, n, dup_every=9)
    for j in rng.choice(n, 12, replace=False):
        L.point(int(j), rng.uniform(X[1, 0], X[-2, 0]), rng.uniform(-2, 2), v=rng.uniform(-0.3, 0.3, 2))
    return Case(f"dynamic_dt{dt}", X, L.types, L.params, dt, ("dynamic",))


def footprint_case(N, seed):
    """random headings, random positions, every third entry a duplicate of an earlier one: the only equal distances are those
    of duplicates, which are equal whatever the distance arithmetic (off the grid, no distance sits on a threshold)"""
    rng = np.random.default_rng(seed)
    X = _dyadic_line_poses(rng, N)
    X[:, 2] = rng.uniform(-np.pi, np.pi, N)
    n = 240
    L = _List(n)
    for j in range(n):
        if j % 3 == 2:
            src = int(rng.integers(0, j)); L.types[j], L.params[j] = L.types[src], L.params[src]
        else:
            L.point(j, rng.uniform(X[1, 0] - 3, X[-2, 0] + 3), rng.uniform(-3, 3))
    return Case(f"footprint_{seed}", X, L.types, L.params, 0.3, ("footprint",))


def overflow_cases(N=24, seeds=(11, 12)):
    """dense grid points along a long horizon: more than 64 distinct selections, so the resident list fills up and drops"""
    out = []
    for s in seeds:
        rng = np.random.default_rng(3000 + s)
        X = _dyadic_line_poses(rng, N, step=0.375)
        L = _dense_points(rng, X, LIST_MAX if s % 2 else 900, spread=1.5, dup_every=5)
        out.append(Case(f"overflow_{s}", X, L.types, L.params, 0.3, ("overflow",)))
    return out


def groups():
    """every case group: (name, configuration, cases)"""
    out = [Group("base", base_cfg(), [ties_and_boundaries()] + list_shapes() + random_poses())]
    for k in (1, 5, 16):
        out.append(Group(f"K{k}", base_cfg(k=k), [forced_cluster(10, k, 24 if k == 16 else 8, 40 + k)]))
    out.append(Group("K0", base_cfg(k=0), [forced_cluster(10, 0, 8, 40), ties_and_boundaries()]))
    lines = base_cfg(); lines.collocation = capi.COLLOC_MIDPOINT
    out.append(Group("typed", lines, [typed_lists()]))
    dyn_fixed = base_cfg(); dyn_fixed.enable_dynamic_obstacles = 1
    out.append(Group("dynamic_fixed_dt", dyn_fixed, [dynamic_list(10, 0.3, 51)]))
    dyn_free = base_cfg(); dyn_free.enable_dynamic_obstacles = 1
    dyn_free.variable_dt, dyn_free.dt_lb, dyn_free.dt_ub = 1, 0.05, 1.0
    out.append(Group("dynamic_free_dt", dyn_free, [dynamic_list(10, 0.4375, 52), dynamic_list(10, 0.1875, 53)]))
    for fp, params, extra in ((capi.FOOTPRINT_CIRCULAR, [0.125, 0, 0, 0], {}),
                              (capi.FOOTPRINT_TWO_CIRCLES, [0.25, 0.125, 0.25, 0.125], {}),
                              (capi.FOOTPRINT_LINE, [-0.25, 0.0, 0.25, 0.0], {}),
                              (capi.FOOTPRINT_POLYGON, None, {})):
        c = base_cfg()
        c.footprint_type = fp
        if params is None:
            c.n_poly = len(configs.CARLIKE_POLYGON)
            for i, (px, py) in enumerate(configs.CARLIKE_POLYGON):
                c.poly_xy[2 * i], c.poly_xy[2 * i + 1] = px, py
        else:
            c.footprint_params[:] = params
        out.append(Group(f"footprint_{fp}", c, [footprint_case(10, 60 + fp), footprint_case(10, 70 + fp)]))
    for k in (8, 16):
        out.append(Group(f"overflow_K{k}", base_cfg(n=24, k=k), overflow_cases()))
    return out


def has_exact_tie(cfg, case, sel):
    """some stage's selection had a competitor at exactly the same distance (a duplicate or a mirror image)"""
    N = case.X.shape[0]
    for k in range(1, N - 1):
        d = [on.footprint_distance(cfg, case.X[k], case.types[j], case.params[j], t=k * case.dt) for j in range(case.count)]
        d = np.array(d)
        for j in sel[:, k]:
            if j >= 0 and (d == d[j]).sum() > 1:
                return True
    return False
