"""ctypes binding of the CPU SIMT-emulation harness (tests/emu/emu.cpp) — test infrastructure only."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
sys.path.insert(0, _ROOT)
from paddlerobotics_b200._config import B2QConfig, OBS_DIM, INFO_DIM  # noqa: E402  (pure-ctypes struct mirror, no CUDA)

_SO = os.path.join(_HERE, "_build", "libb2q_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", _HERE, "-s"])
        _lib = C.CDLL(_SO)
    return _lib


class EmuEnv:
    def __init__(self, n=1, precision=1, **kw):
        self.n = n
        self.dtype = np.float64 if precision else np.float32
        cfg = B2QConfig()
        lib().emu_default_config(C.byref(cfg))
        cfg.num_envs = n
        cfg.precision = precision
        self._keep = None
        for k, v in kw.items():
            if k == "heightfield":
                hf, x0, y0, cell = v
                hf = np.ascontiguousarray(hf, dtype=np.float64)
                self._keep = hf
                cfg.terrain_type = 1
                cfg.hf_ny, cfg.hf_nx = hf.shape
                cfg.hf_x0, cfg.hf_y0, cfg.hf_cell = x0, y0, cell
                cfg.hf_host = hf.ctypes.data_as(C.POINTER(C.c_double))
            elif k == "noise_stdev":
                for i in range(5):
                    cfg.noise_stdev[i] = float(v[i])
            elif k == "base_damping":
                for i in range(4):
                    cfg.base_damping[i] = float(v[i])
            else:
                setattr(cfg, k, v)
        self.cfg = cfg
        self.h = C.c_void_p()
        rc = lib().emu_create(C.byref(cfg), C.byref(self.h))
        assert rc == 0, rc

    def _a(self, x, shape):
        return np.ascontiguousarray(np.asarray(x, dtype=self.dtype).reshape(shape))

    def set_dynamics(self, dyn=None, mask=None):
        d = None if dyn is None else self._a(dyn, (self.n, 48))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        lib().emu_set_dynamics(self.h, None if m is None else m.ctypes.data_as(C.c_void_p), None if d is None else d.ctypes.data_as(C.c_void_p))

    def obs_dim(self):
        return int(lib().emu_obs_dim(self.h))

    def set_force(self, f=None):
        a = None if f is None else self._a(f, (self.n, 3))
        lib().emu_set_force(self.h, None if a is None else a.ctypes.data_as(C.c_void_p))

    def reset(self, etg_w=None, etg_b=None, mask=None, x_offset=None):
        w = None if etg_w is None else self._a(np.broadcast_to(np.asarray(etg_w).reshape(-1, 3, 20), (self.n, 3, 20)), (self.n, 3, 20))
        b = None if etg_b is None else self._a(np.broadcast_to(np.asarray(etg_b).reshape(-1, 3), (self.n, 3)), (self.n, 3))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        obs = np.zeros((self.n, self.obs_dim()), dtype=self.dtype)
        x = None if x_offset is None else self._a(x_offset, (self.n,))
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        lib().emu_reset(self.h, p(m), p(w), p(b), p(x), p(obs))
        return obs

    def step(self, action, donef=False):
        a = self._a(action, (self.n, 60 if int(getattr(self.cfg, 'motor_mode', 0)) == 2 else 12))
        obs = np.zeros((self.n, self.obs_dim()), dtype=self.dtype)
        rew = np.zeros(self.n, dtype=self.dtype)
        done = np.zeros(self.n, dtype=np.uint8)
        info = np.zeros((self.n, INFO_DIM), dtype=self.dtype)
        p = lambda x: x.ctypes.data_as(C.c_void_p)
        lib().emu_step(self.h, p(a), C.c_int(int(donef)), p(obs), p(rew), p(done), p(info))
        return obs, rew, done, info

    def get_state(self):
        s = np.zeros((self.n, 37), dtype=self.dtype)
        lib().emu_get_state(self.h, s.ctypes.data_as(C.c_void_p))
        return s

    def set_state(self, s):
        s = self._a(s, (self.n, 37))
        lib().emu_set_state(self.h, s.ctypes.data_as(C.c_void_p))

    def close(self):
        if self.h:
            lib().emu_destroy(self.h)
            self.h = None


# ---- the step kernel's scalar primitives through their host branches (same call surface as tests/gpu_probe/probe.py)
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _dt(prec):
    return np.float64 if prec else np.float32


def sincos(a):
    a = np.ascontiguousarray(a, dtype=np.float32); s, c = np.zeros_like(a), np.zeros_like(a)
    lib().emu_sincos_f(a.size, _p(a), _p(s), _p(c))
    return s, c


def unary(which, x):
    """m_rcp (0) or m_rsqrt (1) of a float32 array."""
    x = np.ascontiguousarray(x, dtype=np.float32); y = np.zeros_like(x)
    lib().emu_unary_f(which, x.size, _p(x), _p(y))
    return y


def philox4(seeds, ctr):
    seeds = np.ascontiguousarray(seeds, dtype=np.uint64); ctr = np.ascontiguousarray(ctr, dtype=np.uint32).reshape(-1, 3)
    out = np.zeros((seeds.size, 4), dtype=np.uint32)
    lib().emu_philox4(seeds.size, _p(seeds), _p(ctr), _p(out))
    return out


def philox_normal4(prec, seeds, ctr):
    seeds = np.ascontiguousarray(seeds, dtype=np.uint64); ctr = np.ascontiguousarray(ctr, dtype=np.uint32).reshape(-1, 3)
    out = np.zeros((seeds.size, 4), dtype=_dt(prec))
    lib().emu_philox_normal4(prec, seeds.size, _p(seeds), _p(ctr), _p(out))
    return out


def leg(prec, legs, x, inverse):
    legs = np.ascontiguousarray(legs, dtype=np.int32); x = np.ascontiguousarray(x, dtype=_dt(prec)).reshape(-1, 3)
    out = np.zeros_like(x)
    lib().emu_leg(prec, legs.size, int(inverse), _p(legs), _p(x), _p(out))
    return out


def rpy(prec, q):
    q = np.ascontiguousarray(q, dtype=_dt(prec)).reshape(-1, 4); out = np.zeros((q.shape[0], 3), dtype=q.dtype)
    lib().emu_rpy(prec, q.shape[0], _p(q), _p(out))
    return out


def terrain(prec, hf, x0, y0, cell, xy):
    hf = np.ascontiguousarray(hf, dtype=np.float64); xy = np.ascontiguousarray(xy, dtype=_dt(prec)).reshape(-1, 2)
    out = np.zeros((xy.shape[0], 4), dtype=xy.dtype)
    lib().emu_terrain(prec, hf.shape[1], hf.shape[0], C.c_double(x0), C.c_double(y0), C.c_double(cell), _p(hf), xy.shape[0], _p(xy), _p(out))
    return out


def solve(prec, S21, b):
    S21 = np.ascontiguousarray(S21, dtype=_dt(prec)).reshape(-1, 21); b = np.ascontiguousarray(b, dtype=_dt(prec)).reshape(-1, 6)
    x = np.zeros_like(b)
    lib().emu_solve(prec, b.shape[0], _p(S21), _p(b), _p(x))
    return x
