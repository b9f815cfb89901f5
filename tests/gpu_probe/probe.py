"""ctypes binding of the device probe (tests/gpu_probe/probe.cu) — test infrastructure only.

The library is built on first use with the product's nvcc flags into tests/gpu_probe/_build/ and rebuilt when a source it includes is newer.
Every call takes and returns NumPy arrays; the probe copies them through device buffers of its own."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
sys.path.insert(0, _ROOT)
from paddlerobotics_b200 import build as _b  # noqa: E402  (flags and header list only; imports no CUDA)

_SO = os.path.join(_HERE, "_build", "libb2q_probe.so")
_DEPS = [os.path.join(_HERE, f) for f in ("probe.cu", "prim.h")] + [os.path.join(_b.CSRC, h) for h in _b.HEADERS + ["b2q_philox.cuh"]]
_lib = None
NBLK = 132 * 16                     # sweep grid: 16 blocks of 256 threads per H100 SM
PH_N = 8


def build():
    if os.path.exists(_SO) and all(os.path.getmtime(p) <= os.path.getmtime(_SO) for p in _DEPS if os.path.exists(p)):
        return _SO
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = _SO + ".%d.tmp" % os.getpid()
    subprocess.check_call([nvcc] + _b.NVCC_FLAGS + ["-o", tmp, os.path.join(_HERE, "probe.cu")])
    os.replace(tmp, _SO)
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.probe_sweep.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.probe_philox.argtypes = [C.c_uint32, C.c_int, C.c_void_p]
        _lib.probe_terrain.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _ok(rc, what):
    assert rc == 0, "%s: cudaError %d" % (what, rc)


def f32_bits(x):
    return int(np.float32(x).view(np.uint32))


def sweep(which, lo, hi, both):
    """Exhaustive sweep of m_sincos (0), m_rcp (1) or m_rsqrt (2) over the float bit patterns lo..hi (and their negatives when `both`).
    Returns (worst err0, its input, worst err1, its input, flag count); see the ops in probe.cu."""
    err = np.zeros((NBLK, 2)); arg = np.zeros((NBLK, 2), dtype=np.uint32); cnt = np.zeros(NBLK, dtype=np.uint64)
    _ok(lib().probe_sweep(which, lo, hi, int(both), NBLK, _p(err), _p(arg), _p(cnt)), "probe_sweep")
    i0, i1 = int(np.argmax(err[:, 0])), int(np.argmax(err[:, 1]))
    as_f = lambda b: float(np.uint32(b).view(np.float32))
    return float(err[i0, 0]), as_f(arg[i0, 0]), float(err[i1, 1]), as_f(arg[i1, 1]), int(cnt.sum())


def philox(n):
    """Philox over n (key, counter) tuples; a dict of the reductions of k_philox."""
    out = np.zeros((NBLK, PH_N))
    _ok(lib().probe_philox(n, NBLK, _p(out)), "probe_philox")
    return {"word_mismatch": int(out[:, 0].sum()), "normal_mismatch": int(out[:, 1].sum()), "n4f_rel": float(out[:, 2].max()),
            "n4f_abs_exact_u": float(out[:, 3].max()), "n4d_rel": float(out[:, 4].max()), "pn_rel": float(out[:, 5].max()),
            "pn_abs_exact_u": float(out[:, 6].max()), "first_mismatch": float(out[:, 7].min())}


def sincos(a):
    a = np.ascontiguousarray(a, dtype=np.float32); n = a.size
    s, c = np.zeros(n, np.float32), np.zeros(n, np.float32); ds, dc = np.zeros(n), np.zeros(n)
    _ok(lib().probe_sincos(n, _p(a), _p(s), _p(c), _p(ds), _p(dc)), "probe_sincos")
    return s, c, ds, dc


def unary(which, x):
    """m_rcp (0) or m_rsqrt (1) of a float32 array on the device."""
    x = np.ascontiguousarray(x, dtype=np.float32); y = np.zeros_like(x)
    _ok(lib().probe_unary(which, x.size, _p(x), _p(y)), "probe_unary")
    return y


def _dt(prec):
    return np.float64 if prec else np.float32


def leg(prec, legs, x, inverse):
    """leg_fk (toe minus hip joint origin) or leg_inv (leg_ik's joint angles) of [n,3] inputs, leg index per row."""
    legs = np.ascontiguousarray(legs, dtype=np.int32); x = np.ascontiguousarray(x, dtype=_dt(prec)).reshape(-1, 3)
    out = np.zeros_like(x)
    _ok(lib().probe_leg(prec, legs.size, int(inverse), _p(legs), _p(x), _p(out)), "probe_leg")
    return out


def rpy(prec, q):
    q = np.ascontiguousarray(q, dtype=_dt(prec)).reshape(-1, 4); out = np.zeros((q.shape[0], 3), dtype=q.dtype)
    _ok(lib().probe_rpy(prec, q.shape[0], _p(q), _p(out)), "probe_rpy")
    return out


def terrain(prec, hf, x0, y0, cell, xy):
    """[n,4] (height, normal) of terrain_height on the field hf [ny,nx] at [n,2] points."""
    hf = np.ascontiguousarray(hf, dtype=np.float64); xy = np.ascontiguousarray(xy, dtype=_dt(prec)).reshape(-1, 2)
    out = np.zeros((xy.shape[0], 4), dtype=xy.dtype)
    _ok(lib().probe_terrain(prec, hf.shape[1], hf.shape[0], x0, y0, cell, _p(hf), xy.shape[0], _p(xy), _p(out)), "probe_terrain")
    return out


def solve(prec, S21, b):
    S21 = np.ascontiguousarray(S21, dtype=_dt(prec)).reshape(-1, 21); b = np.ascontiguousarray(b, dtype=_dt(prec)).reshape(-1, 6)
    x = np.zeros_like(b)
    _ok(lib().probe_solve(prec, b.shape[0], _p(S21), _p(b), _p(x)), "probe_solve")
    return x
