"""ctypes binding of tests/bezier_host.cpp: the Bezier gait's shared host/device arithmetic (csrc/b2q_bezier.h) compiled for the CPU into a
temporary directory — test infrastructure only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="b2q_bezier_host_"), "libbezier_host.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-shared", "-std=c++17", "-x", "c++", "-ffp-contract=off",
                               "-o", out, os.path.join(_HERE, "bezier_host.cpp")])
        _lib = C.CDLL(out)
        _lib.bez_rollout.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 6
        _lib.bez_ik.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        _lib.bez_state_dim.restype = C.c_int
    return _lib


def rollout(q, contact):
    """q [n,12] reset joint angles, contact [n,steps] bits of the reference foot -> tb0 [n,4,3], feet [n,steps,4,3], ang [n,steps,12],
    flags [n,steps,3] = (TD, SwRef, StanceSwing)."""
    q = np.ascontiguousarray(q, dtype=np.float64).reshape(-1, 12)
    n = q.shape[0]
    c = np.ascontiguousarray(contact, dtype=np.uint8).reshape(n, -1)
    steps = c.shape[1]
    tb0, feet = np.empty((n, 12)), np.empty((n, steps, 12))
    ang, flags = np.empty((n, steps, 12)), np.empty((n, steps, 3))
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().bez_rollout(n, steps, p(q), p(c), p(tb0), p(feet), p(ang), p(flags))
    return tb0.reshape(n, 4, 3), feet.reshape(n, steps, 4, 3), ang, flags


def ik(feet):
    """feet [..., 4, 3] in the base frame -> the A1 IK joint angles [..., 12] (NaN for an unreachable foot)."""
    f = np.ascontiguousarray(feet, dtype=np.float64)
    out = np.empty(f.shape[:-2] + (12,))
    lib().bez_ik(int(f.size // 12), f.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out
