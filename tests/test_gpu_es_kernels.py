"""The ES kernels of csrc/b2q_es.cu, called through the C ABI, against the plain restatements of tests/es_ref.py at training shapes and at
the edges where a kernel goes wrong: block boundaries, the fitness kernel's strided loop (rollouts > 32), NaN and inf inputs, and every
exit of the ETG fit's gradient-descent loop.  es_accumulate, es_fitness, dyn_accumulate and dyn_finish must match bit for bit in both
precisions; every output buffer is followed by a guard region that must come back untouched."""
import ctypes as C

import numpy as np
import pytest

import es_ref as R

pytestmark = pytest.mark.gpu

GUARD = 300                                   # elements after each output buffer: more than a 256-thread block


@pytest.fixture(scope="module")
def lib():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from paddlerobotics_b200 import _lib
    return _lib.load()


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Guarded:
    """A device buffer with `GUARD` sentinel elements after its end: .t is the buffer, check() asserts that the guard is unchanged."""

    def __init__(self, host, sentinel):
        import torch
        host = np.ascontiguousarray(host)
        full = np.concatenate([host.reshape(-1), np.full(GUARD, sentinel, host.dtype)])
        self.buf = torch.from_numpy(full).cuda()
        self.guard = self.buf[host.size:].clone()
        self.t = self.buf[:host.size].view(host.shape)

    def ptr(self):
        return self.t.data_ptr()

    def host(self):
        return self.t.cpu().numpy()

    def check(self):
        import torch
        g = self.buf[self.t.numel():]
        b = torch.uint8
        assert torch.equal(g.view(b), self.guard.view(b)), "write past the end of the buffer"


def _sentinel(dtype):
    return {np.float32: np.float32(np.nan), np.float64: np.nan, np.int32: np.int32(0x5EADBEEF), np.uint8: np.uint8(0xA5)}[np.dtype(dtype).type]


def G(host):
    return Guarded(host, _sentinel(host.dtype))


def assert_bits(got, want):
    """Equal bit for bit, except that any NaN matches any NaN (the GPU returns the canonical NaN, the host keeps the operand's payload)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype
    if got.dtype.kind == "f":
        gn, wn = np.isnan(got), np.isnan(want)
        assert np.array_equal(gn, wn), np.nonzero(gn != wn)
        iv = got.dtype.str.replace("f", "i")
        bad = np.nonzero(got[~gn].view(iv) != want[~wn].view(iv))[0]
        assert bad.size == 0, (bad[:5], got[~gn][bad[:5]], want[~wn][bad[:5]])
    else:
        assert np.array_equal(got, want), np.nonzero(got != want)


DTYPES = {4: np.float32, 8: np.float64}


# ---- b2q_es_accumulate
@pytest.mark.parametrize("es", [4, 8])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 65537])
def test_es_accumulate_bit_exact(lib, es, n):
    """Eight control steps.  Env kinds by e % 4: done on the first step, done on every step from the second, never done, random done.
    NaN and +-inf rewards are placed after each env's first done (they must not reach ret) and before or at it in some envs (they must).
    Some envs start dead; ret and len start from nonzero values."""
    dt = DTYPES[es]
    rng = np.random.default_rng(n * 10 + es)
    steps = 8
    reward = (rng.standard_normal((steps, n)) * 10.0 ** rng.uniform(-2, 2, (steps, n))).astype(dt)
    kind = np.arange(n) % 4
    done = np.zeros((steps, n), np.uint8)
    done[0, kind == 0] = 1
    done[1:, kind == 1] = 7                                           # any nonzero byte is done
    done[:, kind == 3] = rng.random((steps, int((kind == 3).sum()))) < 0.3
    alive0 = np.ones(n, np.uint8)
    alive0[(np.arange(n) % 11 == 5)] = 0                              # already finished before this window
    first = np.where(done.any(0), done.argmax(0), steps)
    poison = np.array([np.nan, np.inf, -np.inf], dt)
    for e in range(n):
        if first[e] + 1 < steps:                                      # after done: must stay out of ret
            reward[first[e] + 1:, e] = poison[np.arange(steps - first[e] - 1) % 3]
    before = (np.arange(n) % 13 == 2) & (first >= 1)                  # before done (or never done): must reach ret
    reward[0, before] = poison[np.arange(int(before.sum())) % 3]
    at = (np.arange(n) % 17 == 0)                                     # on the done step itself: still accumulated
    reward[np.minimum(first[at], steps - 1), np.nonzero(at)[0]] = np.nan
    ret0 = rng.standard_normal(n).astype(dt)
    len0 = rng.integers(0, 50, n).astype(np.int32)

    ret, ln, alive = G(ret0), G(len0), G(alive0)
    rew_d = [G(reward[k]) for k in range(steps)]
    done_d = [G(done[k]) for k in range(steps)]
    r_ret, r_len, r_alive = ret0.copy(), len0.copy(), alive0.copy()
    for k in range(steps):
        assert lib.b2q_es_accumulate(rew_d[k].ptr(), done_d[k].ptr(), alive.ptr(), ret.ptr(), ln.ptr(), n, es, _stream()) == 0
        R.es_accumulate(r_ret, r_len, r_alive, reward[k], done[k])
    assert_bits(ret.host(), r_ret)
    assert_bits(ln.host(), r_len)
    assert_bits(alive.host(), r_alive)
    for g in (ret, ln, alive):
        g.check()
    if n > 1:                                                         # the cases the test is about occurred
        assert np.isnan(r_ret).any() and np.isinf(r_ret).any() and np.isfinite(r_ret).any()
        assert (r_alive == 0).any() and (r_alive == 1).any()


# ---- b2q_es_fitness
@pytest.mark.parametrize("es", [4, 8])
@pytest.mark.parametrize("pop", [1, 3, 4, 5, 257])
def test_es_fitness_bit_exact(lib, es, pop):
    """rollouts 1 .. 100, including 31 / 32 / 33 around the warp width and 64 / 100 where every lane sums two or more rollouts in the
    strided loop; returns spanning six decades so that a different summation order changes the last bits; mean_len NULL and not."""
    dt = DTYPES[es]
    for rollouts in (1, 2, 16, 31, 32, 33, 64, 100):
        rng = np.random.default_rng(pop * 1000 + rollouts + es)
        n = pop * rollouts
        ret = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(dt)
        length = rng.integers(0, 100000, n).astype(np.int32)
        want_f, want_l = R.es_fitness(ret, length, pop, rollouts)
        ret_d, len_d = G(ret), G(length)
        for with_len in (False, True):
            fit = G(np.zeros(pop, dt))
            ml = G(np.zeros(pop, dt)) if with_len else None
            assert lib.b2q_es_fitness(ret_d.ptr(), len_d.ptr(), fit.ptr(), ml.ptr() if ml else None, pop, rollouts, es, _stream()) == 0
            assert_bits(fit.host(), want_f)
            fit.check()
            if ml:
                assert_bits(ml.host(), want_l)
                ml.check()
        assert np.array_equal(ret_d.host(), ret) and np.array_equal(len_d.host(), length)    # inputs untouched


# ---- b2q_dyn_accumulate / b2q_dyn_finish
@pytest.mark.parametrize("es", [4, 8])
@pytest.mark.parametrize("steps", [1, 100])
@pytest.mark.parametrize("n", [1, 17, 18, 4096, 65537])
def test_dyn_accumulate_and_finish_bit_exact(lib, es, steps, n):
    """n = 18 is where n x 15 threads first cross one 256-thread block.  Every info column the kernel must not read holds NaN, and the
    columns it reads get new values each step, with per-step statistics."""
    import torch
    dt = DTYPES[es]
    rng = np.random.default_rng(n + steps + es)
    info = torch.full((n, 56), float("nan"), dtype=torch.float32 if es == 4 else torch.float64, device="cuda")
    acc = G(np.zeros((n, 15), dt))
    ref = np.zeros((n, 15), dt)
    scale = 10.0 ** rng.uniform(-1, 1, (1, 15))
    for t in range(steps):
        x = (rng.standard_normal((n, 15)) * scale).astype(dt)
        mean = (rng.standard_normal(15) * scale[0] * 0.3).astype(dt)
        std = rng.uniform(0.05, 1.0, 15).astype(dt)
        info[:, 42:54] = torch.from_numpy(x[:, :12]).cuda()
        info[:, 39:42] = torch.from_numpy(x[:, 12:]).cuda()
        m_d, s_d = G(mean), G(std)
        assert lib.b2q_dyn_accumulate(info.data_ptr(), m_d.ptr(), s_d.ptr(), acc.ptr(), n, es, _stream()) == 0
        R.dyn_accumulate(ref, x, mean, std)
    got = acc.host()
    assert_bits(got, ref)
    assert np.isfinite(got).all()
    acc.check()
    rew = G(np.zeros(n, dt))
    assert lib.b2q_dyn_finish(acc.ptr(), steps, rew.ptr(), n, es, _stream()) == 0
    assert_bits(rew.host(), R.dyn_finish(ref, steps))
    rew.check()


@pytest.mark.parametrize("es", [4, 8])
def test_dyn_finish_propagates_nan_and_inf(lib, es):
    """A NaN in a single accumulated column, in the motor group or in the drpy group and at every position, makes the reward NaN (the
    reference's np.max propagates NaN; a NaN-dropping max returned a finite reward computed from the other 14 columns).  +inf in a
    single column makes it -inf.  Rows without them stay finite and bit-exact."""
    dt = DTYPES[es]
    rng = np.random.default_rng(es)
    acc = np.abs(rng.standard_normal((64, 15))).astype(dt)
    for c in range(15):
        acc[2 * c, c] = np.nan
        acc[2 * c + 1, c] = np.inf
    acc_d, rew = G(acc), G(np.zeros(64, dt))
    assert lib.b2q_dyn_finish(acc_d.ptr(), 7, rew.ptr(), 64, es, _stream()) == 0
    got = rew.host()
    rew.check()
    assert np.isnan(got[0:30:2]).all(), got[0:30:2]
    assert (got[1:30:2] == -np.inf).all(), got[1:30:2]
    assert np.isfinite(got[30:]).all()
    assert_bits(got, R.dyn_finish(acc, 7))


# ---- b2q_etg_fit
def _etg_inputs(golden):
    from paddlerobotics_b200.etg import ETG_layer
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    A = np.array([layer.update(t) for t in [0.35, 0, 0.05, 0.1, 0.15, 0.2]]).reshape(6, 20)
    return A, golden["opt_points"], golden["opt_w0"], golden["opt_b0"]


def _device_fit(lib, A, pp, sols, w0, b0, lamb, precision):
    import torch
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")
    pop = sols.shape[0]
    w, b = G(np.zeros((pop, 3, 20))), G(np.zeros((pop, 3)))
    o, p_, s_, w0_, b0_ = t(A), t(pp), t(sols.reshape(pop, 12)), t(w0), t(b0)
    assert lib.b2q_etg_fit(o.data_ptr(), p_.data_ptr(), s_.data_ptr(), w0_.data_ptr(), b0_.data_ptr(), float(lamb), float(precision),
                           w.ptr(), b.ptr(), pop, _stream()) == 0
    out = w.host(), b.host()
    w.check(); b.check()
    return out


def _check_fit(w_dev, b_dev, A, pp, sols, w0, b0, lamb, precision, tol=1e-9):
    """w_dev [pop, 3, 20] against the host iteration: rows 0 and 2 are the x and z solves, row 1 is zero; b is (b0[0], 0, b0[2]) exactly.
    The device thread must stop where the host loop stops; where the host's residual at the exit step (or the one before it) lies within
    1e-9 (relative) of `precision`, a device whose rounding put it on the other side of `precision` may stop one iteration later (or
    earlier), and that iterate is accepted too.  Non-finite entries must be non-finite exactly where the host's are."""
    pop = sols.shape[0]
    pts = pp[None] + sols.reshape(pop, 6, 2)
    assert np.array_equal(b_dev, np.repeat(np.array([[b0[0], 0.0, b0[2]]]), pop, 0))
    assert np.array_equal(w_dev[:, 1], np.zeros((pop, 20)))
    ties, iters_all = 0, []
    for row, col in ((0, 0), (2, 1)):
        B = (pts[:, :, col] - b0[row]).T
        xs, errs, iters = R.ls_sol_batch(A, B, w0[row], precision, lamb=lamb)
        iters_all.append(iters)
        for p in range(pop):
            k = int(iters[p])
            cands = [k]
            near = lambda e: abs(e - precision) <= 1e-9 * abs(precision)
            if k < 1000 and near(errs[k, p]):
                cands.append(k + 1)
            if k > 0 and near(errs[k - 1, p]):
                cands.append(k - 1)
            ties += len(cands) > 1
            got = w_dev[p, row]
            ok = False
            for c in cands:
                want = xs[c, :, p]
                fin = np.isfinite(want)
                if np.array_equal(fin, np.isfinite(got)) and np.abs(got[fin] - want[fin]).max(initial=0) <= tol:
                    ok = True
                    break
            assert ok, (row, p, k, cands, np.abs(got - xs[k, :, p]).max())
    return np.concatenate(iters_all), ties


@pytest.mark.parametrize("pop", [1, 31, 33, 256])
def test_etg_fit_matches_the_host_iteration_over_ga_generations(lib, golden, pop):
    """SimpleGA draws at sigma 0.02 (the ETG ES phase's) and 0.1, over three generations (ask / tell with the draws' own spread as
    fitness), with the reference's lamb 0.5 and precision 1e-4: w within 1e-9 of the host iterate at the host's exit step, b exact."""
    from paddlerobotics_b200.es import SimpleGA
    A, pp, w0, b0 = _etg_inputs(golden)
    iters = []
    for sigma in (0.02, 0.1):
        np.random.seed(pop + int(sigma * 100))
        ga = SimpleGA(12, sigma_init=sigma, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=max(0.1, 1.0 / pop), weight_decay=0.005, popsize=pop,
                      param=np.zeros(12))                      # at least one elite, so that later generations can be drawn
        for gen in range(3):
            sols = ga.ask()
            w, b = _device_fit(lib, A, pp, sols, w0, b0, 0.5, 1e-4)
            it, _ = _check_fit(w, b, A, pp, sols, w0, b0, 0.5, 1e-4)
            iters.append(it)
            ga.tell(-np.abs(sols).sum(1))
    iters = np.concatenate(iters)
    assert (iters == 1000).any()
    if pop >= 31:
        assert (iters < 1000).any()              # both of the loop's exits ran


def test_etg_fit_loop_exits(lib, golden):
    """precision 0: every solve runs exactly 1000 iterations.  precision above the starting residual: no iteration, w == w0 exactly.
    lamb 100: gradient descent diverges (step factor about 4); the device's w is non-finite exactly where the host's is."""
    from paddlerobotics_b200.es import SimpleGA
    A, pp, w0, b0 = _etg_inputs(golden)
    np.random.seed(7)
    sols = SimpleGA(12, sigma_init=0.02, popsize=33, param=np.zeros(12)).ask()
    w, b = _device_fit(lib, A, pp, sols, w0, b0, 0.5, 0.0)
    it, _ = _check_fit(w, b, A, pp, sols, w0, b0, 0.5, 0.0)
    assert (it == 1000).all()
    w, b = _device_fit(lib, A, pp, sols, w0, b0, 0.5, 1e6)
    it, _ = _check_fit(w, b, A, pp, sols, w0, b0, 0.5, 1e6)
    assert (it == 0).all()
    assert np.array_equal(w[:, 0], np.repeat(w0[None, 0], 33, 0)) and np.array_equal(w[:, 2], np.repeat(w0[None, 2], 33, 0))
    w, b = _device_fit(lib, A, pp, sols, w0, b0, 100.0, 1e-4)
    it, _ = _check_fit(w, b, A, pp, sols, w0, b0, 100.0, 1e-4)
    assert not np.isfinite(w[:, 0]).any() and (it < 1000).all()
