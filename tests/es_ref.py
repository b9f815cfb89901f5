"""Plain restatements of the ES and replay-memory kernels (csrc/b2q_es.cu, csrc/b2q_rpm.cu) for the tests.

es_accumulate, es_fitness, dyn_accumulate and dyn_finish have no multiply-add pairs and divide with IEEE division (the library is built
without --use_fast_math), so restated in the kernel's own operation order and precision they give the device's result bit for bit.
ls_sol is etg.LS_sol with its iteration count and error trace; ls_sol_batch runs the same iteration for a whole population at once and
keeps every iterate, so that a test can pick the one at which a device thread must have stopped.  rpm_slots is the replay sampler's
slot formula in wrapping uint64 arithmetic."""
from copy import copy

import numpy as np

DYN_MOTOR, DYN_DRPY = 42, 39          # info columns of the 12 joint angles and of the 3 body rates (obs-IMU[3:]), include/b2q.h


def es_accumulate(ret, length, alive, reward, done):
    """One control step of b2q_es_accumulate, in place: for alive envs ret += reward, len += 1, and alive is cleared on done."""
    a = alive != 0
    ret[a] = ret[a] + reward[a]
    length[a] += 1
    alive[a & (done != 0)] = 0


def es_fitness(ret, length, pop, rollouts):
    """b2q_es_fitness in the kernel's order: lane l of individual i sums ret[i, r] for r = l, l + 32, ... in that order (from 0), the lanes
    are combined by the xor butterfly s += s[lane ^ o] for o = 16, 8, 4, 2, 1, and lane 0's sum is divided by `rollouts`.  The lengths
    likewise, converted to ret's type.  Returns (fitness [pop], mean_len [pop])."""
    t = ret.dtype.type
    out = []
    for x in (ret.reshape(pop, rollouts), length.reshape(pop, rollouts).astype(ret.dtype)):
        k = -(-rollouts // 32)
        pad = np.zeros((pop, 32 * k), ret.dtype)      # s + 0 == s: the padding adds nothing, and s is never -0
        pad[:, :rollouts] = x
        s = np.zeros((pop, 32), ret.dtype)
        for j in range(k):
            s = s + pad[:, 32 * j:32 * (j + 1)]
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, lane ^ o]
        out.append(s[:, 0] / t(rollouts))
    return out[0], out[1]


def dyn_columns(info):
    """The 15 values b2q_dyn_accumulate reads from info [n, 56]: joint angles (columns 42-53), then body rates (39-41)."""
    return np.concatenate([info[:, DYN_MOTOR:DYN_MOTOR + 12], info[:, DYN_DRPY:DYN_DRPY + 3]], axis=1)


def dyn_accumulate(acc, x15, mean15, std15):
    """acc [n, 15] += (x - mean)^2 / std^2, in the kernel's order: d = x - mean; acc + (d * d) / (s * s)."""
    d = x15 - mean15[None, :]
    s = std15[None, :]
    acc[...] = acc + (d * d) / (s * s)


def dyn_finish(acc, steps):
    """reward [n] = 30 - (max_j acc[:, j] / steps + max_k acc[:, 12 + k] / steps) / 2, the maxima taken left to right with np.maximum,
    which propagates NaN as the reference's np.max does."""
    t = acc.dtype.type
    lm, ld = acc[:, 0], acc[:, 12]
    for c in range(1, 12):
        lm = np.maximum(lm, acc[:, c])
    for c in range(13, 15):
        ld = np.maximum(ld, acc[:, c])
    return t(30) - (lm / t(steps) + ld / t(steps)) / t(2)


def ls_sol(A, b, precision=1e-4, alpha=0.05, lamb=1, w0=None):
    """etg.LS_sol (ETGRL/train.py:59-79) with the same operations, returning (x, iterations, errors): errors[k] is the squared residual
    after k iterations, and the loop ran while errors[k] > precision, at most 1000 times."""
    n, m = A.shape
    x = copy(w0) if w0 is not None else np.zeros((m, 1))
    err = A.dot(x) - b
    err = err.transpose().dot(err)
    errs = [err.item()]
    i = 0
    while err > precision and i < 1000:
        A1 = A.transpose().dot(A)
        dx = A1.dot(x) - A.transpose().dot(b)
        if w0 is not None:
            dx += lamb * (x - w0)
        x = x - alpha * dx
        err = A.dot(x) - b
        err = err.transpose().dot(err)
        errs.append(err.item())
        i += 1
    return x, i, np.array(errs)


def ls_sol_batch(A, B, w0, precision, alpha=0.05, lamb=0.5):
    """The ls_sol iteration for many right-hand sides at once: B [6, pop], w0 [20].  Every column runs the full 1000 iterations (a
    column's iterates do not depend on the others), so xs[k] [20, pop] and errs[k] [pop] are the iterate and squared residual after k
    iterations and iters[p] is where ls_sol stops: the first k with not errs[k] > precision, else 1000."""
    w0 = np.asarray(w0, np.float64).reshape(-1, 1)
    AtA, Atb = A.T.dot(A), A.T.dot(B)
    x = np.repeat(w0, B.shape[1], axis=1)
    xs, errs = [x], []
    with np.errstate(over="ignore", invalid="ignore"):
        r = A.dot(x) - B
        errs.append((r * r).sum(0))
        for _ in range(1000):
            x = x - alpha * (AtA.dot(x) - Atb + lamb * (x - w0))
            r = A.dot(x) - B
            xs.append(x)
            errs.append((r * r).sum(0))
    xs, errs = np.array(xs), np.array(errs)
    running = errs[:1000] > precision                    # NaN > precision is False: a non-finite residual ends the loop
    iters = np.where(running.all(0), 1000, np.argmin(running, axis=0))
    return xs, errs, iters


# ---- replay sampler (rpm_sample_kernel / rpm_sample_cursor_kernel)
_U = np.uint64


def rpm_mix(x):
    """splitmix64 finaliser, upper 32 bits (as uint64)."""
    x = np.asarray(x, dtype=np.uint64)
    x = x + _U(0x9E3779B97F4A7C15)
    x = (x ^ (x >> _U(30))) * _U(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> _U(27))) * _U(0x94D049BB133111EB)
    x = x ^ (x >> _U(31))
    return x >> _U(32)


def rpm_slots(seed, batch, size):
    """Ring slots of a sample of `batch` rows from [0, size): slot_i = (mix(seed * 0x100000001B3 + i) * size) >> 32, in wrapping uint64.
    The device cursor's sample uses seed + state[2] as `seed`."""
    key = np.array([seed], dtype=np.uint64) * _U(0x100000001B3) + np.arange(batch, dtype=np.uint64)
    return ((rpm_mix(key) * _U(size)) >> _U(32)).astype(np.int64)
