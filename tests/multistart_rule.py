"""The multistart selection rule (mpcb200_step_batch_multistart) restated in numpy, and the ranking of the bumped lines of the cold
start: the test-side statements the device selection and the oracle / emulator initial guesses are checked against."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np

from mpc_local_planner_b200 import capi

BUMP_STEP = 0.4
BUMP_MARGIN = 0.05


def winner(status, obj, inf, hysteresis):
    """Candidate index of one robot's winner.  status / obj / inf: [K] per candidate (0: the incumbent); a status < 0 (an unfinished
    solve) counts as MAX_ITER."""
    st = [capi.STATUS_MAX_ITER if s < 0 else int(s) for s in status]
    K = len(st)
    conv = [k for k in range(1, K) if st[k] == capi.STATUS_CONVERGED]
    cs = None
    for k in conv:   # least objective, the lower k on ties
        if cs is None or obj[k] < obj[cs]:
            cs = k
    if st[0] == capi.STATUS_CONVERGED:
        if cs is None:
            return 0
        return cs if obj[cs] < obj[0] - (1.0 - hysteresis) * abs(obj[0]) else 0
    if cs is not None:
        return cs
    stopped = (capi.STATUS_MAX_ITER, capi.STATUS_MAX_TIME)
    if st[0] in stopped:
        return 0
    best = 0
    for k in range(1, K):
        if st[k] in stopped and (best == 0 or inf[k] < inf[best]):
            best = k
    return best


def winners_from_scal(scal, B, K, hysteresis):
    """winner of every robot from the SCAL words of the B*K slots ([B*K, SCAL_WORDS], candidate k of robot b in row k*B + b)"""
    out = np.zeros(B, dtype=np.int32)
    for b in range(B):
        rows = scal[[k * B + b for k in range(K)]]
        out[b] = winner(rows[:, capi.SC_STATUS], rows[:, capi.SC_OBJ], rows[:, capi.SC_INF], hysteresis)
    return out


def ranking(scores, margin=1e-9):
    """Indices of the lines (m + n for m = -n..n) in rank order: repeated selection, a line beats the best so far only when its
    score is below best - margin (1 + best), the lower m first."""
    left = list(range(len(scores)))
    order = []
    while left:
        best, bi = 1e300, None
        for i in left:
            if scores[i] < best - margin * (1.0 + best):
                best, bi = scores[i], i
        order.append(bi)
        left.remove(bi)
    return order


def straight(cfg, data, b, orc):
    """the straight line start -> goal of instance b (the cold start without obstacles)"""
    o = orc.Instance(cfg, data["x0"][b], data["xf"][b])
    o.init_cold()
    return o.arr("X").copy()


def scores(cfg, data, b, orc, Xs):
    """score of every bumped line m = -n..n: 1e-3 |A| + the clearance violation of its interior stages"""
    cnt, types, params = data["obstacles"]
    n, N = cfg.initial_guess_bumps, int(cfg.n)
    xf, x0 = data["xf"][b], data["x0"][b]
    nv = np.array([-(xf[1] - x0[1]), xf[0] - x0[0]]); nv /= np.linalg.norm(nv)
    out = []
    for m in range(-n, n + 1):
        A = BUMP_STEP * m
        s = 1e-3 * abs(A)
        for k in range(1, N - 1):
            o = A * math.sin(math.pi * k / (N - 1))
            pose = np.array([Xs[0, k] + o * nv[0], Xs[1, k] + o * nv[1], Xs[2, k]])
            for j in range(cnt[b]):
                op = np.ascontiguousarray(params[b, j])
                d = orc.lib().orc_footprint_distance(C.byref(cfg), orc._dp(pose), int(types[b, j]), orc._dp(op), None, None)
                s += max(0.0, cfg.min_obstacle_dist + BUMP_MARGIN - d)
        out.append(s)
    return np.array(out), nv


def line_of(X, Xs, nv, N):
    """m of the bumped line whose positions X holds (lateral offset at the middle stage)"""
    k = (N - 1) // 2
    off = float(np.dot(X[:2, k] - Xs[:2, k], nv)) / math.sin(math.pi * k / (N - 1))
    m = round(off / BUMP_STEP)
    assert abs(off - BUMP_STEP * m) < 1e-9
    return m


def clear_ranks(scores, order):
    """ranks whose line's score is not within twice the decision margin of another line's"""
    ok = []
    for r, i in enumerate(order):
        s = scores[i]
        if all(abs(scores[j] - s) > 2e-9 * (1.0 + abs(s)) for j in order if j != i):
            ok.append(r)
    return ok


# ---- the ranked cold initial guess of the oracle and of the emulator: tests/multistart/*.{c,cpp} on top of the two, compiled with
#      the flags of their makefiles into a directory of this process ----
_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


def _native(name):
    if name not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="mpcb200_multistart_"), name + ".so")
        if name == "ranked_oracle":
            cmd = [os.environ.get("CC", "gcc"), "-O3", "-march=x86-64-v3", "-fPIC", "-std=gnu11", "-shared", "-o", out,
                   os.path.join(_HERE, "multistart", "ranked_oracle.c"), "-lm", "-lpthread"]
        else:
            cmd = [os.environ.get("CXX", "g++"), "-O2", "-march=x86-64-v3", "-fPIC", "-std=c++17", "-shared", "-o", out,
                   os.path.join(_HERE, "multistart", "ranked_emu.cpp"), "-lm"]
        subprocess.check_call(cmd, stdout=subprocess.DEVNULL)
        lib = C.CDLL(out)
        if name == "ranked_oracle":
            lib.orc_init_cold_rank.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
            lib.orc_init_cold_rank.restype = None
        else:
            lib.emu_init_cold_rank.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_int]
            lib.emu_init_cold_rank.restype = None
        _LIBS[name] = lib
    return _LIBS[name]


def oracle_init_cold_rank(inst, rank):
    """cold initial guess of an oracle Instance (oracle_py) from the bumped line of rank `rank`; rank 0 is inst.init_cold()"""
    _native("ranked_oracle").orc_init_cold_rank(C.addressof(inst.p), int(rank), C.cast(inst.ws, C.c_void_p))


def emu_init_cold_rank(inst, rank):
    """cold initial guess of an emulator EmuInstance (emu_py) from the bumped line of rank `rank`: init(force_cold=True) with a rank"""
    _native("ranked_emu").emu_init_cold_rank(C.addressof(inst.cfg), inst.W.ctypes.data_as(C.POINTER(C.c_double)), int(rank))
