"""ctypes binding of the CPU warp emulator (tests/emu/libemu.so) -- TEST INFRASTRUCTURE.  It replays the device code
(the same host/device headers the CUDA kernels are compiled from) for one instance on the CPU."""
import ctypes as C
import os
import subprocess

import numpy as np

from mpc_local_planner_b200 import capi

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "libemu.so")
_LIB = None


def build(force=False):
    srcs = [os.path.join(_DIR, "emu.cpp")] + [
        os.path.join(_DIR, "..", "..", "mpc_local_planner_b200", "csrc", f)
        for f in ("mpc_core.h", "mpc_stage.h", "mpc_riccati_warp.h", "mpc_layout.h")]
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(LIB_PATH) < os.path.getmtime(s) for s in srcs if os.path.exists(s)):
        subprocess.check_call(["make", "-C", _DIR, "-B", "libemu.so"], stdout=subprocess.DEVNULL)


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            build()
        L = C.CDLL(LIB_PATH)
        cp, dp, ip = C.POINTER(capi.Config), C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.emu_stride.restype = C.c_longlong
        L.emu_stride.argtypes = [cp]
        L.emu_field_offset.argtypes = [cp, C.c_int, ip]
        L.emu_scatter.argtypes = [cp, dp, dp, dp, dp, C.c_int, ip, dp, C.c_int, dp, dp, C.c_int]
        L.emu_scatter.restype = None
        L.emu_reset.argtypes = [cp, dp]
        L.emu_init.argtypes = [cp, dp, C.c_int]
        L.emu_associate.argtypes = [cp, dp, C.c_double, C.c_int]
        L.emu_eval.argtypes = [cp, dp, C.c_double]
        L.emu_kkt.argtypes = [cp, dp]
        L.emu_linesearch.argtypes = [cp, dp, C.c_double]
        L.emu_solve.argtypes = [cp, dp, C.c_double, C.c_int]
        L.emu_outputs.argtypes = [cp, dp, dp, dp]
        L.emu_resample.argtypes = [C.c_int, dp, dp, C.c_double, C.c_int, dp, dp]
        L.emu_resample.restype = C.c_double
        L.emu_vp_stage.argtypes = [cp, dp, ip]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def resample(X, U, dt, n_new):
    X = np.ascontiguousarray(X, dtype=np.float64); U = np.ascontiguousarray(U, dtype=np.float64)
    Xn = np.zeros((3, n_new)); Un = np.zeros((2, n_new))
    dt_new = lib().emu_resample(X.shape[1], _dp(X), _dp(U), float(dt), int(n_new), _dp(Xn), _dp(Un))
    return Xn, Un, dt_new


class EmuInstance:
    def __init__(self, cfg, x0, xf, u_prev=(0.0, 0.0), u_prev_dt=0.0, obst_types=None, obst_params=None, vp=None,
                 x_init=None):
        self.L = lib()
        self.cfg = cfg.copy()
        self.N = int(cfg.n)
        self.u_prev_dt = float(u_prev_dt)
        self.W = np.zeros(int(self.L.emu_stride(C.byref(self.cfg))))
        self._inputs = None
        self.set_inputs(x0, xf, u_prev, obst_types, obst_params, vp, x_init)
        self.L.emu_reset(C.byref(self.cfg), _dp(self.W))

    def set_inputs(self, x0, xf, u_prev=(0.0, 0.0), obst_types=None, obst_params=None, vp=None, x_init=None, reinit=0):
        x0 = np.ascontiguousarray(x0, dtype=np.float64)
        xf = np.ascontiguousarray(xf, dtype=np.float64)
        up = np.ascontiguousarray(u_prev, dtype=np.float64)
        ot = np.ascontiguousarray(obst_types if obst_types is not None else np.zeros(0), dtype=np.int32)
        op = np.ascontiguousarray(obst_params if obst_params is not None else np.zeros((0, 5)), dtype=np.float64)
        v = np.ascontiguousarray(vp if vp is not None else np.zeros((0, 3)), dtype=np.float64)
        xi = np.ascontiguousarray(x_init, dtype=np.float64) if x_init is not None else None
        self.L.emu_scatter(C.byref(self.cfg), _dp(self.W), _dp(x0), _dp(xf), _dp(up), int(ot.shape[0]),
                           ot.ctypes.data_as(C.POINTER(C.c_int)), _dp(op), int(v.shape[0]), _dp(v), _dp(xi), int(reinit))

    def field(self, f):
        cnt = C.c_int()
        off = self.L.emu_field_offset(C.byref(self.cfg), f, C.byref(cnt))
        if f == capi.F_SCAL:
            return self.W[off: off + cnt.value]
        if f == capi.F_KKT:  # stage records [k][43] (42 words + a zero word); present [42][N] (copy)
            idx = off + np.arange(self.N)[None, :] * 43 + np.arange(cnt.value)[:, None]
            return self.W[idx]
        if f == capi.F_OBSIDX:  # one signed byte per (slot, stage)
            return self.W[off:].view(np.int8)[: cnt.value * self.N].reshape(cnt.value, self.N).astype(np.float64)
        return self.W[off: off + cnt.value * self.N].reshape(cnt.value, self.N)

    def set_field(self, f, a):
        """write a workspace field in the layout field(f) returns (F_KKT: [42][N] into the stage records)"""
        cnt = C.c_int()
        off = self.L.emu_field_offset(C.byref(self.cfg), f, C.byref(cnt))
        a = np.asarray(a, dtype=np.float64)
        if f == capi.F_SCAL:
            self.W[off: off + cnt.value] = a
        elif f == capi.F_KKT:
            idx = off + np.arange(self.N)[None, :] * 43 + np.arange(cnt.value)[:, None]
            self.W[idx] = a
        elif f == capi.F_OBSIDX:
            raise ValueError("OBSIDX is written by the association only")
        else:
            self.W[off: off + cnt.value * self.N] = a.reshape(-1)

    def vp_stage(self, n_vp):
        """the stages the association gave the first n_vp via-points"""
        out = np.zeros(64, dtype=np.int32)
        V = self.L.emu_vp_stage(C.byref(self.cfg), _dp(self.W), out.ctypes.data_as(C.POINTER(C.c_int)))
        assert n_vp <= V
        return out[:n_vp].copy()

    def init(self, force_cold=False):
        self.L.emu_init(C.byref(self.cfg), _dp(self.W), int(force_cold))

    def associate(self, first_outer=True):
        self.L.emu_associate(C.byref(self.cfg), _dp(self.W), self.u_prev_dt, int(first_outer))

    def eval(self):
        return self.L.emu_eval(C.byref(self.cfg), _dp(self.W), self.u_prev_dt)

    def kkt(self):
        return self.L.emu_kkt(C.byref(self.cfg), _dp(self.W))

    def linesearch(self):
        self.L.emu_linesearch(C.byref(self.cfg), _dp(self.W), self.u_prev_dt)

    def solve(self, force_cold=False):
        return self.L.emu_solve(C.byref(self.cfg), _dp(self.W), self.u_prev_dt, int(force_cold))

    def outputs(self):
        u = np.empty((self.N, 2))
        x = np.empty((self.N, 3))
        self.L.emu_outputs(C.byref(self.cfg), _dp(self.W), _dp(u), _dp(x))
        return u, x


def instance_from_batch(cfg, data, b, x_init=None):
    cnt, types, params = data["obstacles"] if data.get("obstacles") is not None else (None, None, None)
    ot = types[b, : cnt[b]] if cnt is not None else None
    op = params[b, : cnt[b]] if cnt is not None else None
    vp = None
    if data.get("viapoints") is not None:
        vc, vposes = data["viapoints"]
        vp = vposes[b, : vc[b]]
    return EmuInstance(cfg, data["x0"][b], data["xf"][b], data["u_prev"][b], data["u_prev_dt"], ot, op, vp, x_init)
