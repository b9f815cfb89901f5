"""The float32 product kernel (the one the benchmark and training run), through the C ABI, against the float64 oracle: every feature
switch, every terrain preset with make_env's feature set, full warps of different robots, in-step auto-reset, masked reset and
set_dynamics, the CTA size and the height-field far edges.  Teacher-forced (tests/f32_cases.py): before every step the oracle state is
loaded into the kernel, so each comparison measures one control step's float32 error.

Each bound is about 4x the largest error measured on an H100 80GB HBM3 (700 W power limit) over seeds 0-2; the measured value sits
beside it.  Relative errors are scaled by max(1, |reference|_inf); contact flags, done and the fall flag are bit-exact."""
import numpy as np
import pytest

import f32_cases as F

pytestmark = pytest.mark.gpu

# case -> (bound on the relative obs / q-dot / reward / info error, measured worst over seeds 0-2)
BOUNDS = {
    "noise": (2.6e-4, 6.6e-5), "torque": (1.0e-4, 2.3e-5), "hybrid_filter": (2.9e-4, 7.3e-5), "joint_limits": (1.2e-4, 3.1e-5),
    "knee_jlim_body": (5.0e-2, 1.2e-2), "push_damping": (1.9e-4, 4.6e-5), "filter_interp_clip": (5.4e-4, 1.4e-4), "latency": (1.7e-4, 4.3e-5),
    "layout_raw_units": (2.6e-4, 6.6e-5), "layout_subset": (2.6e-4, 6.6e-5),
    "make_env_stairstair": (2.7e-4, 6.6e-5), "make_env_slopeslope": (1.6e-4, 4.1e-5), "make_env_stairslope": (2.7e-4, 6.6e-5),
    "make_env_slopestair": (1.6e-4, 4.1e-5), "make_env_terrain": (1.9e-4, 4.8e-5), "make_env_balancebeam": (3.3e-4, 8.3e-5),
}
# Why most bounds sit above 1e-4: obs carries the joint angles as (q - pose) / 0.1 and rpy x 10, so a 1e-5 joint-angle error is a 1e-4
# observation error.  Every bound above 1e-4 is also held to the oracle's own conditioning: on every step and measure,
# error <= EXCESS x (the oracle's response to f32-rounded inputs on that step) + F.FLOOR.  Measured multiples: at most 122 on flat
# ground, 157 on the stairs, 249 on the knee case (a contact that switches on between substeps) and 376 on the balance beam.  The
# likely reason the terrain cases sit higher (not proven here): a one-cell riser is a slope of 4 in the bilinear field and the beam's
# edge a slope of 15, so the f32 rounding of the foot position inside its cell moves the contact height by that slope times the
# rounding, while on the flat plane height and normal are exact.  The input-rounding sensitivity does not contain that rounding, which
# happens inside the step.
# Re-measured with the sensitivity clone's observation history carried forward from step to step (f32_cases.teacher_forced): the
# multiples are unchanged (seed 0 on the H100: 122 flat, 157 stairs, 249 knees, 107 mixed), because no case held to this rule has a
# control latency that reaches back into the previous control step (the latency case is 12 ms, the mixed-robot rows 0 ms).
EXCESS = 1600.0


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch


def _np(t):
    return t.detach().double().cpu().numpy()


class _Gpu:
    """VecQuadrupedalEnv with float64 numpy in / out, for the teacher-forced runner."""

    def __init__(self, env):
        self.env = env

    def set_state(self, s):
        self.env.set_state(s)

    def get_state(self):
        return _np(self.env.get_state())

    def step(self, a):
        ob, rw, dn, inf = self.env.step(a)
        return _np(ob), _np(rw), dn.cpu().numpy(), _np(inf)


def _gait(name, etg_stable, etg_default, etg_shipped):
    return dict(stable=etg_stable, default=etg_default, shipped=etg_shipped)[name]


def run_case(name, seed, w, b, precision="f32"):
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    gait, kw, kind, steps, hf, row, xo, force, knee_rest = F.case_inputs(name)
    env = VecQuadrupedalEnv(1, precision=precision, heightfield=hf, **kw)
    if row is not None:
        env.set_dynamics(row[None, :])
    ob0 = _np(env.reset(w, b, x_offset=None if xo is None else [xo]))[0]
    o, oo = F.make_oracle(kw, hf, w, b, row, xo, force)
    if force is not None:
        env.set_external_force(np.asarray(force)[None, :])
    rng = np.random.default_rng(seed)
    rec = F.teacher_forced(_Gpu(env), [o], [F.actions(kind, rng, k, 1) for k in range(steps)], F.flag_columns(kw), knee_rest)
    env.close()
    return ob0, oo, rec


def check(name, rec, bound):
    print(F.summary(name, rec))
    for k, i, err, sens, mm in rec:
        assert mm is None, (name, k, i, mm)
    assert F.worst(rec)[0] <= bound, (name, F.worst(rec))
    if bound > 1e-4:
        for k, i, err, sens, mm in rec:
            for m in F.METRICS:
                assert err[m] <= EXCESS * sens[m] + F.FLOOR, (name, k, i, m, err[m], sens[m])


@pytest.mark.parametrize("name", list(F.CASES))
def test_f32_teacher_forced_per_feature(torch_cuda, etg_stable, etg_default, etg_shipped, name):
    """One case per feature switch (noise, TORQUE, HYBRID with the filter switched on, joint limits driven into the stops, knee
    contacts, push + damping, filter + interpolation + command clip, a control latency of several substeps, two reduced sensor layouts)
    and make_env's feature set on every terrain preset, started just before the obstacle."""
    w, b = _gait(F.CASES[name][0], etg_stable, etg_default, etg_shipped)
    ob0, oo, rec = run_case(name, 0, w, b)
    assert np.abs(ob0 - oo).max() / max(1.0, np.abs(oo).max()) < 1e-4, name       # reset observation (f32 settle vs f64 settle)
    check(name, rec, BOUNDS[name][0])


def test_f32_sensor_noise_statistics(torch_cuda, etg_stable):
    """float32 Box-Muller on the GPU: the difference between a noisy and a clean handle driven identically is zero-mean Gaussian with
    the configured stdev per channel (motor angle, velocity, rpy, rpy rate), independent across envs."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    n, steps = 64, 12
    noisy = VecQuadrupedalEnv(n, noise_stdev=F.NOISE, noise_seed=12345)
    clean = VecQuadrupedalEnv(n)
    noisy.reset(w, b); clean.reset(w, b)
    z = np.zeros((n, 12), np.float32)
    d = {"q": [], "qd": [], "rpy": [], "drpy": []}
    for k in range(steps):
        on = _np(noisy.step(z)[0]); oc = _np(clean.step(z)[0])
        d["q"].append((on[:, 13:25] - oc[:, 13:25]) * 0.1)          # obs = (q - pose) / 0.1
        d["qd"].append(on[:, 25:37] - oc[:, 25:37])
        d["rpy"].append((on[:, 7:10] - oc[:, 7:10]) * 0.1)
        d["drpy"].append((on[:, 10:13] - oc[:, 10:13]) * 0.5)
    for key, s in (("q", F.NOISE[0]), ("qd", F.NOISE[1]), ("rpy", F.NOISE[3]), ("drpy", F.NOISE[4])):
        x = np.concatenate(d[key]).ravel() / s
        kurt = ((x - x.mean()) ** 4).mean() / x.var() ** 2
        print("noise %-4s  samples %5d  std/s %.4f  mean/s %+.4f  kurtosis %.3f" % (key, x.size, x.std(), x.mean(), kurt))
        assert abs(x.std() - 1) < 0.06 and abs(x.mean()) < 0.06 and abs(kurt - 3) < 0.4, (key, x.std(), x.mean(), kurt)
    per_env = np.stack(d["qd"])[:, :, 0]                               # one channel over time, per env: the streams differ between envs
    assert len({tuple(np.round(per_env[:, i], 6)) for i in range(n)}) == n
    noisy.close(); clean.close()


def test_f32_mixed_robots_full_warps(torch_cuda, etg_shipped):
    """N = 21: two full warps (8 robots each) and a ragged one.  Every env has its own dynamics row, x offset and actions; only some
    drive into the joint stops or onto their knees, so the warp-uniform general solve runs for robots that do not need it.  Teacher-forced,
    each env against its own oracle."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_shipped
    n = 21
    rng = np.random.default_rng(21)
    kw = dict(F.MAKE_ENV_FEATS)
    rows = np.stack([_row(rng, latency=0.0) for _ in range(n)])
    xo = rng.uniform(-0.1, 0.1, n)
    kinds = ["stops" if i % 5 == 2 else "knees" if i % 7 == 4 else "residual" for i in range(n)]
    env = VecQuadrupedalEnv(n, **kw)
    env.set_dynamics(rows)
    env.reset(w, b, x_offset=xo)
    oracles = [F.make_oracle(kw, None, w, b, rows[i], xo[i], env_id=i)[0] for i in range(n)]
    acts = []
    for k in range(10):
        a = np.concatenate([F.actions(kinds[i], rng, k, 1) for i in range(n)])
        acts.append(a)
    rec = F.teacher_forced(_Gpu(env), oracles, acts, F.flag_columns(kw), knee_rest=True)
    env.close()
    walk = [r for r in rec if kinds[r[1]] == "residual"]
    down = [r for r in rec if kinds[r[1]] != "residual"]
    print(F.summary("mixed: walking robots", walk)); print(F.summary("mixed: stops / knees", down))
    check("mixed_walking", walk, MIXED_BOUND)                  # robots that share their warp with the general solve but need none
    for k, i, err, sens, mm in down:                           # robots crashing onto their knees: held to the oracle's conditioning only
        assert mm is None, (k, i, mm)
        for m in F.METRICS:
            assert err[m] <= EXCESS * sens[m] + F.FLOOR, (k, i, kinds[i], m, err[m], sens[m])


MIXED_BOUND = 2.9e-4               # measured 7.2e-5 on this seed (the stops / knees robots: at most 107x their sensitivity)


def _row(rng, latency=None):
    """A dynamics row drawn as the reference's param2dynamic_dict does, with the foot friction pinned to 0.8 (as the f64 random-dynamics
    tests pin it) so that these tests keep their measured plain bounds: sticking feet make a step ill-conditioned and raise the f32 error
    several-fold.  The full friction range, 0 to 10.2, is covered under the conditioning rule by tests/test_gpu_full_range.py.  (The 400x
    excess once seen here at friction 3 was the 37-43 ms latency of these rows reading the previous step's substeps, see
    f32_cases.teacher_forced, not a float32 defect.)"""
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    d = param2dynamic_dict(rng.uniform(-0.3, 0.3, 48))
    d["footfriction"] = 0.8
    if latency is not None:
        d["control_latency"] = latency
    return dynamic_dict_to_row(d)


def _batch_oracles(ob):
    """OracleEnv views of an OracleBatch's envs (get_state / set_state on the batch's own structs)."""
    from oracle import oracle as O
    views = []
    for i in range(ob.n):
        v = O.OracleEnv.__new__(O.OracleEnv)
        v.cfg, v.e = ob.cfg, ob.envs[i]
        views.append(v)
    return views


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("n", [13, 40])
def test_in_step_auto_reset_vs_oracle_batch(torch_cuda, etg_default, precision, n):
    """In-step auto-reset over falls (default gait, +-0.3 residuals) against OracleBatch(auto_reset=True).  float64 runs free; float32
    is teacher-forced (the oracle state is loaded before every step), and after a fall both sides restart from their own settled
    snapshot."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    env = VecQuadrupedalEnv(n, precision=precision, auto_reset=True)
    env.reset(w, b)
    ob = O.OracleBatch(n, etg_w=w, etg_b=b)
    views = _batch_oracles(ob)
    rng = np.random.default_rng(n)
    tol = 1e-7 if precision == "f64" else AUTO_RESET_BOUND
    ndone = worst = 0.0
    for k in range(50):
        if precision == "f32":
            env.set_state(np.stack([v.get_state() for v in views]))
        a = rng.uniform(-0.3, 0.3, (n, 12))
        o1, r1, d1, i1 = (_np(x) for x in env.step(a))
        o2, r2, d2, i2 = ob.step(a, auto_reset=True)
        assert np.array_equal(d1.astype(bool), d2.astype(bool)), (k, np.nonzero(d1 != d2))
        assert np.array_equal(o1[:, 3:7], o2[:, 3:7]) and np.array_equal(i1[:, F.FALL], i2[:, F.FALL]), k
        for x, y in ((o1, o2), (r1[:, None], r2[:, None]), (i1, i2)):
            e = (np.abs(x - y).max(1) / np.maximum(1.0, np.abs(y).max(1))).max()
            worst = max(worst, e)
            assert e <= tol, (k, e)
        ndone += int(d2.sum())
    print("auto-reset %s n=%d: %d resets, worst rel %.3g" % (precision, n, ndone, worst))
    assert ndone >= 3
    env.close()


AUTO_RESET_BOUND = 2.6e-4          # measured 6.5e-5 (n = 40)


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_masked_reset_and_set_dynamics(torch_cuda, etg_stable, precision):
    """Masked reset and masked set_dynamics: masked envs equal a fresh oracle reset (with their new dynamics row); unmasked envs'
    state and observation rows are bit-identical to before the call, and all go on matching their oracles."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    n = 21
    rng = np.random.default_rng(3)
    rows = np.stack([_row(rng) for _ in range(n)])
    env = VecQuadrupedalEnv(n, precision=precision)
    env.set_dynamics(rows)
    xo = rng.uniform(-0.1, 0.1, n)
    env.reset(w, b, x_offset=xo)
    oracles = [F.make_oracle({}, None, w, b, rows[i], xo[i], env_id=i)[0] for i in range(n)]
    eng = _Gpu(env)
    tol = 1e-7 if precision == "f64" else MASK_BOUND

    def run(steps):
        rec = F.teacher_forced(eng, oracles, [rng.uniform(-0.2, 0.2, (n, 12)) for _ in range(steps)], F.flag_columns({}))
        assert all(r[4] is None for r in rec) and F.worst(rec)[0] <= tol, F.worst(rec)
        return F.worst(rec)[0]

    def masked(call, mask, fresh):
        st0, ob0 = _np(env.get_state()), _np(env.obs)
        call()
        st1, ob1 = _np(env.get_state()), _np(env.obs)
        assert np.array_equal(st1[~mask], st0[~mask]) and np.array_equal(ob1[~mask], ob0[~mask])
        for i in np.nonzero(mask)[0]:
            o, oo = fresh(i)
            oracles[i] = o
            assert np.abs(ob1[i] - oo).max() / max(1.0, np.abs(oo).max()) < (1e-9 if precision == "f64" else 1e-4), i
            # f32: the settled snapshot of a randomised robot lies up to 1.1e-4 (measured) from the f64 one
            assert np.abs(st1[i] - o.get_state()).max() < (1e-10 if precision == "f64" else 4.5e-4), i

    e1 = run(6)
    m1 = np.arange(n) % 3 == 0
    xo2 = rng.uniform(-0.1, 0.1, n)
    masked(lambda: env.reset(w, b, env_mask=m1, x_offset=xo2), m1, lambda i: F.make_oracle({}, None, w, b, rows[i], xo2[i], env_id=i))
    e2 = run(6)
    m2 = np.arange(n) % 4 == 1
    rows2 = rows.copy()
    rows2[m2] = np.stack([_row(rng) for _ in range(int(m2.sum()))])
    st0, ob0 = _np(env.get_state()), _np(env.obs)
    env.set_dynamics(rows2, env_mask=m2)
    assert np.array_equal(_np(env.get_state())[~m2], st0[~m2]) and np.array_equal(_np(env.obs), ob0)
    masked(lambda: env.reset(w, b, env_mask=m2, x_offset=xo2), m2, lambda i: F.make_oracle({}, None, w, b, rows2[i], xo2[i], env_id=i))
    e3 = run(6)
    print("masked reset / set_dynamics %s: worst rel %.3g %.3g %.3g" % (precision, e1, e2, e3))
    env.close()


MASK_BOUND = 2.3e-4                # measured 5.8e-5 on this seed


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("n", [13, 40, 4096])
def test_cta_size_bit_identical(torch_cuda, etg_default, precision, n):
    """threads_per_block 32, 64 and 128 on the default (non-FEAT) path: the per-robot arithmetic does not depend on the CTA size, so
    obs, reward, done, info and state are bit-identical, through falls and in-step auto-resets."""
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    g = torch.Generator(device="cuda"); g.manual_seed(n)
    dt = torch.float32 if precision == "f32" else torch.float64
    acts = [torch.rand(n, 12, device="cuda", generator=g, dtype=dt) * 0.6 - 0.3 for _ in range(30)]
    outs = []
    for tpb in (32, 64, 128):
        env = VecQuadrupedalEnv(n, precision=precision, auto_reset=True, threads_per_block=tpb)
        env.reset(w, b, x_offset=torch.linspace(-0.1, 0.1, n))
        res, ndone = [], 0
        for a in acts:
            ob, rw, dn, inf = env.step(a)
            res.append((ob.clone(), rw.clone(), dn.clone(), inf.clone()))
            ndone += int(dn.sum())
        res.append((env.get_state(),))
        outs.append(res)
        env.close()
        assert ndone > 0
    for other in outs[1:]:
        for x, y in zip(outs[0], other):
            assert all(torch.equal(p, q) for p, q in zip(x, y))


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("where", list(F.EDGE_CASES))
def test_heightfield_far_edges(torch_cuda, etg_stable, precision, where):
    """A sloped 40 x 40 field whose far x / y edge lies behind the robot's feet, exactly under the front / left toes, and one cell past
    them.  In float32, nx - 1.000001 rounds to nx - 1, so the lookup must clamp the cell index as an integer: an unclamped index reads
    the next row's first column (x) or past the end of the field (y)."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    hf = F.sloped_field(*F.EDGE_CASES[where])
    env = VecQuadrupedalEnv(1, precision=precision, heightfield=hf)
    ob0 = _np(env.reset(w, b))[0]
    o, oo = F.make_oracle({}, hf, w, b)
    tol = 1e-9 if precision == "f64" else 1e-4
    assert np.abs(ob0 - oo).max() / max(1.0, np.abs(oo).max()) < tol, where
    rng = np.random.default_rng(4)
    rec = F.teacher_forced(_Gpu(env), [o], [rng.uniform(-0.2, 0.2, (1, 12)) for _ in range(8)], F.flag_columns({}))
    env.close()
    print(F.summary("edge_%s_%s" % (where, precision), rec))
    assert all(r[4] is None for r in rec)
    assert F.worst(rec)[0] <= (1e-7 if precision == "f64" else EDGE_BOUND), F.worst(rec)


EDGE_BOUND = 2.3e-4                # measured 5.7e-5
