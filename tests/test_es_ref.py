"""The restatements in tests/es_ref.py, checked on the host against the reference's own numbers: they are what the GPU tests of the ES
and replay kernels compare the device with (tests/test_gpu_es_kernels.py, tests/test_gpu_replay_kernels.py)."""
import numpy as np
import pytest
from scipy import stats

import es_ref as R

EPS64 = np.finfo(np.float64).eps / 2          # unit roundoff


def _etg_system():
    from paddlerobotics_b200.etg import ETG_layer
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    return np.array([layer.update(t) for t in [0.35, 0, 0.05, 0.1, 0.15, 0.2]]).reshape(6, 20)


def test_dyn_restatement_gives_the_reference_loss(golden):
    """Fed the golden recording, the accumulate / finish restatement gives 30 - loss_func(...) of Dynamic_parallel_model.py:29-41, which
    the golden file holds as the reference function's own output.  The reference takes np.mean (pairwise sum) where the kernel sums
    step by step: the two agree to float64 rounding of a 100-term sum of non-negative terms."""
    motor, drpy = golden["dynloss_motor"], golden["dynloss_drpy"]
    mean = np.concatenate([golden["dynloss_exp_motor_mean"], golden["dynloss_exp_drpy_mean"]], 1)
    std = np.concatenate([golden["dynloss_exp_motor_std"], golden["dynloss_exp_drpy_std"]], 1)
    steps = motor.shape[0]
    info = np.full((steps, 56), np.nan)
    info[:, 42:54], info[:, 39:42] = motor, drpy
    acc = np.zeros((1, 15))
    for t in range(steps):
        R.dyn_accumulate(acc, R.dyn_columns(info[t:t + 1]), mean[t], std[t])
    got = R.dyn_finish(acc, steps)[0]
    want = 30.0 - float(golden["dynloss_value"])
    bound = 4 * steps * EPS64 * (30.0 + acc.max() / steps)
    assert abs(got - want) <= bound, (got, want, bound)
    assert got != 30.0 and np.isfinite(got)


def test_dyn_finish_restatement_propagates_nan_and_inf():
    acc = np.abs(np.random.default_rng(0).standard_normal((4, 15)))
    acc[1, 5] = np.nan                 # motor group
    acc[2, 13] = np.nan                # drpy group
    acc[3, 0] = np.inf
    r = R.dyn_finish(acc, 10)
    assert np.isfinite(r[0]) and np.isnan(r[1]) and np.isnan(r[2]) and r[3] == -np.inf


def test_ls_sol_trace_equals_etg_ls_sol_and_opt_with_points(golden):
    """ls_sol returns exactly etg.LS_sol's x, and through it exactly Opt_with_points' weights, on SimpleGA draws at the GA's sigma; its
    error trace is the loop's: every entry before the last is above `precision`, and the last is not (or the loop hit its cap)."""
    from paddlerobotics_b200.es import SimpleGA
    from paddlerobotics_b200.etg import ETG_layer, LS_sol, Opt_with_points
    A = _etg_system()
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w0, b0, pp = golden["opt_w0"], golden["opt_b0"], golden["opt_points"]
    np.random.seed(1)
    sols = SimpleGA(12, sigma_init=0.02, popsize=12, param=np.zeros(12)).ask()
    iters = []
    for sol in sols:
        pts = pp + sol.reshape(6, 2)
        w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, w0=w0, b0=b0, points=pts)
        pt = pts - np.array([b0[0], b0[-1]])
        for col, row in ((0, 0), (1, 2)):
            rhs, x0 = pt[:, col].reshape(-1, 1), w0[row].reshape(-1, 1)
            x, it, errs = R.ls_sol(A, rhs, precision=1e-4, alpha=0.05, lamb=0.5, w0=x0)
            assert np.array_equal(x, LS_sol(A, rhs, precision=1e-4, alpha=0.05, lamb=0.5, w0=x0))
            assert np.array_equal(x.reshape(-1), w[row])
            assert len(errs) == it + 1 and (errs[:-1] > 1e-4).all() and (it == 1000 or not errs[-1] > 1e-4)
            iters.append(it)
    assert 1000 in iters and min(iters) < 1000        # both exits are taken
    x, it, errs = R.ls_sol(A, pt[:, 0].reshape(-1, 1), precision=np.inf, lamb=0.5, w0=w0[0].reshape(-1, 1))
    assert it == 0 and np.array_equal(x.reshape(-1), w0[0]) and len(errs) == 1


@pytest.mark.parametrize("case", ["ga", "capped", "diverging"])
def test_ls_sol_batch_follows_ls_sol(golden, case):
    """The batched iteration stops where ls_sol stops and its iterate there equals ls_sol's x to float64 rounding (it multiplies in another
    order), also when gradient descent diverges (lamb = 100: step factor about 4, so x overflows and the residual ends as NaN)."""
    from paddlerobotics_b200.es import SimpleGA
    A = _etg_system()
    np.random.seed(2)
    sols = SimpleGA(12, sigma_init=0.1 if case == "ga" else 0.02, popsize=16, param=np.zeros(12)).ask()
    w0, b0, pp = golden["opt_w0"], golden["opt_b0"], golden["opt_points"]
    precision, lamb = {"ga": (1e-4, 0.5), "capped": (0.0, 0.5), "diverging": (1e-4, 100.0)}[case]
    B = (pp[None] + sols.reshape(-1, 6, 2))[:, :, 0].T - b0[0]
    xs, errs, iters = R.ls_sol_batch(A, B, w0[0], precision, lamb=lamb)
    for p in range(B.shape[1]):
        with np.errstate(over="ignore", invalid="ignore"):
            x, it, e = R.ls_sol(A, B[:, p:p + 1], precision=precision, lamb=lamb, w0=w0[0].reshape(-1, 1))
        assert it == iters[p]
        xb = xs[it, :, p]
        x = x.reshape(-1)
        fin = np.isfinite(x)
        assert np.array_equal(fin, np.isfinite(xb))
        assert np.abs(xb[fin] - x[fin]).max(initial=0) <= 1e-12 * (1 + np.abs(x[fin]).max(initial=0))
    if case == "capped":
        assert (iters == 1000).all()
    if case == "diverging":
        assert not np.isfinite(xs[iters, :, np.arange(len(iters))]).any() and (iters < 1000).all()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("rollouts", [1, 2, 16, 31, 32, 33, 64, 100, 1000])
def test_tree_order_fitness_is_the_mean_to_rounding(dtype, rollouts):
    """The kernel's sum passes every term through at most ceil(rollouts / 32) - 1 sequential and 5 butterfly additions, then one
    division: |fitness - mean| <= gamma_d * sum|x| / rollouts + u |mean| with d = ceil(rollouts / 32) + 4 (Higham's tree-sum bound)."""
    rng = np.random.default_rng(rollouts)
    pop = 7
    ret = (rng.standard_normal(pop * rollouts) * 10.0 ** rng.uniform(-3, 3, pop * rollouts)).astype(dtype)
    length = rng.integers(0, 1001, pop * rollouts).astype(np.int32)
    fit, mlen = R.es_fitness(ret, length, pop, rollouts)
    assert fit.dtype == dtype and mlen.dtype == dtype
    u = np.finfo(dtype).eps / 2
    d = -(-rollouts // 32) + 4
    gamma = d * u / (1 - d * u)
    x = ret.astype(np.float64).reshape(pop, rollouts)
    mean = x.mean(1)
    bound = gamma * np.abs(x).sum(1) / rollouts + u * np.abs(mean) * 1.0001
    assert (np.abs(fit - mean) <= bound).all(), (np.abs(fit - mean) / bound).max()
    lm = length.reshape(pop, rollouts).astype(np.float64).mean(1)
    assert (np.abs(mlen - lm) <= gamma * lm + u * lm * 1.0001).all()


def test_es_accumulate_restatement_freezes_at_the_first_done():
    ret, ln, alive = np.zeros(3, np.float32), np.zeros(3, np.int32), np.ones(3, np.uint8)
    for r, d in (([1, 2, 3], [1, 0, 0]), ([np.nan, 2, np.inf], [0, 1, 0]), ([np.nan, np.nan, 1], [0, 0, 0])):
        R.es_accumulate(ret, ln, alive, np.array(r, np.float32), np.array(d, np.uint8))
    assert ret[0] == 1 and ret[1] == 4 and ret[2] == np.inf and ln.tolist() == [1, 2, 3] and alive.tolist() == [0, 0, 1]


@pytest.mark.parametrize("size", [1, 2, 3, 1000, 2 ** 20 + 7])
def test_rpm_slots_are_in_range_and_uniform(size):
    """2^20 draws: every slot in [0, size), and the counts pass a chi-square test of uniformity (p > 1e-4)."""
    draws = 2 ** 20
    for seed in (0, 12345, 2 ** 64 - 1):
        s = R.rpm_slots(seed, draws, size)
        assert s.min() >= 0 and s.max() < size
        if size == 1:
            continue
        counts = np.bincount(s, minlength=size)
        exp = draws / size
        chi = ((counts - exp) ** 2 / exp).sum()
        assert stats.chi2.sf(chi, size - 1) > 1e-4, (seed, chi, size)
        assert stats.chi2.cdf(chi, size - 1) > 1e-4, (seed, chi, size)     # not suspiciously even either


def test_rpm_slots_of_consecutive_seeds_are_independent():
    """Seeds s and s + 1 (the sample counter's step): their slot sequences are uncorrelated, equal only as often as chance makes them, and
    their joint distribution over 16 x 16 cells is uniform."""
    n, size = 2 ** 16, 1000
    for s in (0, 1, 999, 2 ** 40):
        a, b = R.rpm_slots(s, n, size), R.rpm_slots(s + 1, n, size)
        assert abs(np.corrcoef(a, b)[0, 1]) < 5 / np.sqrt(n)
        eq = (a == b).sum()
        assert abs(eq - n / size) < 6 * np.sqrt(n / size)
        cells = np.bincount((a * 16 // size) * 16 + b * 16 // size, minlength=256)
        chi = ((cells - n / 256) ** 2 / (n / 256)).sum()
        assert stats.chi2.sf(chi, 255) > 1e-4


def test_rpm_slots_pin_known_values():
    """The formula itself, for a few keys computed by hand from the splitmix64 constants (guards the restatement against edits)."""
    x = (0 * 0x100000001B3 + 0 + 0x9E3779B97F4A7C15) % 2 ** 64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) % 2 ** 64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) % 2 ** 64
    x ^= x >> 31
    assert int(R.rpm_slots(0, 1, 1000)[0]) == ((x >> 32) * 1000) >> 32
    key = (7 * 0x100000001B3 + 5) % 2 ** 64
    x = (key + 0x9E3779B97F4A7C15) % 2 ** 64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) % 2 ** 64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) % 2 ** 64
    x ^= x >> 31
    assert int(R.rpm_slots(7, 6, 2 ** 20 + 7)[5]) == ((x >> 32) * (2 ** 20 + 7)) >> 32
