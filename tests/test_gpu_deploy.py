"""Deployment rehearsal on the GPU: b2q_deploy_obs / b2q_deploy_act against a NumPy restatement bit for bit (both precisions, per-env
step counters, NaN past the table, records, argument errors, CUDA-graph replay), the table-driven control law against the training env's
in-kernel ETG in float64, the shipped student and CPG stair table end to end through deploy_test, and the per-group batch bookkeeping."""
import ctypes as C
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
STUDENT = os.path.join(GOLDEN, "StairStair3_BC1_itr_500383.pt")
CPG = os.path.join(GOLDEN, "gait_action_list_CPG_stairstair7_12_3.npy")
SHIPPED = os.path.join(ROOT, "paddlerobotics_b200", "data", "etg_shipped_gait.npz")
# EnvWrapper.py:50-55
ETG_MEAN = np.array([2.1505982e-02, 3.6674485e-02, -6.0444288e-02, 2.4625482e-02, 1.5869144e-02, -3.2513142e-02, 2.1506395e-02,
                     3.1869926e-02, -6.0140789e-02, 2.4625063e-02, 1.1628972e-02, -3.2163858e-02])
ETG_STD = np.array([4.5967497e-02, 2.0340437e-01, 3.7410179e-01, 4.6187632e-02, 1.9441207e-01, 3.9488649e-01,
                    4.5966785e-02, 2.0323379e-01, 3.7382501e-01, 4.6188373e-02, 1.9457331e-01, 3.9302582e-01])


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _step_counts(env):
    import torch
    sc = torch.empty(env.num_envs, dtype=torch.int32, device=env.device)
    assert env.lib.b2q_get_step_count(env.h, sc.data_ptr(), _stream()) == 0
    return sc.cpu().numpy()


def _env(n, precision, **kw):
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    return VecQuadrupedalEnv(n, precision=precision, etg_enabled=0, **kw)


def _staggered(env, rng):
    """Envs whose step counters differ: every env steps 3 times, the odd ones are reset, then 0..4 more steps per env group."""
    import torch
    n = env.num_envs
    env.reset()
    a = torch.as_tensor(rng.uniform(-0.1, 0.1, (n, 12)), dtype=env.dtype, device=env.device)
    for _ in range(3):
        env.step(a)
    env.reset(env_mask=(np.arange(n) % 2 == 1))
    for k in range(4):
        env.reset(env_mask=(np.arange(n) % 5 == k))      # env groups restart at different steps
        env.step(a)
    return _step_counts(env)


def _np_obs(obs0, sc, table, etg_col, normal, npdt):
    out = obs0.copy()
    mean, istd = ETG_MEAN.astype(npdt), (1.0 / ETG_STD).astype(npdt)
    for e, r in enumerate(sc):
        v = table[r].astype(npdt) if r < len(table) else np.full(12, np.nan, npdt)
        if normal:
            v = (v - mean) * istd
        if etg_col >= 0:
            out[e, etg_col:etg_col + 12] = v
    return out


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("normal", [0, 1])
@pytest.mark.parametrize("sensors", [{}, {"sensor_dis": 0}, {"sensor_etg": 0}, {"sensor_imu": 2, "sensor_motor": 2}])
def test_kernels_against_numpy(precision, normal, sensors):
    """Rows by each env's own step counter (envs reset at different steps), normal 0 / 1, etg_col = -1, the records, and NaN for a
    counter past the table: obs and action equal the NumPy restatement bit for bit."""
    import torch
    from paddlerobotics_b200 import deploy
    npdt = np.float32 if precision == "f32" else np.float64
    rng = np.random.default_rng(7)
    env = _env(37, precision, obs_normal=normal, **sensors)
    sc = _staggered(env, rng)
    assert len(set(sc.tolist())) >= 4 and sc.max() >= 5
    rows = 5                                                        # counters 5 and up lie past the table
    table = rng.uniform(-0.3, 0.3, (rows, 12)).astype(npdt)
    tab = torch.as_tensor(table, device="cuda")
    obs = torch.as_tensor(rng.normal(size=(37, env.observation_dim)).astype(npdt), device="cuda")
    obs0 = obs.cpu().numpy()
    rec_obs = torch.full((9, env.observation_dim), -7.0, dtype=env.dtype, device="cuda")
    etg_col = deploy.etg_col_of(env)
    assert etg_col == (env.observation_dim - 12 if sensors.get("sensor_etg", 1) else -1)
    deploy.deploy_obs(env, tab, rows, obs, rec_obs)
    want = _np_obs(obs0, sc, table, etg_col, normal, npdt)
    got = obs.cpu().numpy()
    assert np.array_equal(got, want, equal_nan=True)
    if etg_col >= 0:
        assert np.isnan(got[sc >= rows, etg_col:]).all() and np.isfinite(got[sc < rows]).all()
    rec_want = np.full((9, env.observation_dim), -7.0, npdt)
    rec_want[sc[0]] = want[0]
    assert np.array_equal(rec_obs.cpu().numpy(), rec_want, equal_nan=True)

    pol = torch.as_tensor(rng.uniform(-1, 1, (37, 12)).astype(np.float32), device="cuda")
    action = torch.full((37, 12), -9.0, dtype=env.dtype, device="cuda")
    rec_act = torch.full((9, 12), -7.0, dtype=env.dtype, device="cuda")
    deploy.deploy_act(env, pol, 0.3, tab, rows, action, rec_act)
    p = pol.cpu().numpy().astype(npdt)
    want_a = np.stack([npdt(0.3) * p[e] + table[r] if r < rows else np.full(12, np.nan, npdt) for e, r in enumerate(sc)])
    assert want_a.dtype == npdt
    assert np.array_equal(action.cpu().numpy(), want_a, equal_nan=True)
    rec_a = np.full((9, 12), -7.0, npdt); rec_a[sc[0]] = want_a[0]
    assert np.array_equal(rec_act.cpu().numpy(), rec_a, equal_nan=True)
    # a record row past rec_rows is not written
    small = torch.full((1, 12), -7.0, dtype=env.dtype, device="cuda")
    if sc[0] >= 1:
        deploy.deploy_act(env, pol, 0.3, tab, rows, action, small)
        assert (small.cpu().numpy() == -7.0).all()
    env.close()


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_table_of_the_kernels_own_etg_gives_the_etg_mode_observation(precision):
    """On an ETG-mode handle, a table whose row k is the kernel's own ETG output at step k (info ETG_act) rewrites the observation's ETG
    block with the bits it already holds."""
    import torch
    from paddlerobotics_b200 import deploy
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    z = np.load(SHIPPED)
    env = VecQuadrupedalEnv(16, precision=precision)
    env.reset(z["w"], z["b"])
    for k in range(7):
        obs, _, _, info = env.step(torch.zeros(16, 12, dtype=env.dtype, device="cuda"))
    table = torch.zeros(8, 12, dtype=env.dtype, device="cuda")
    table[7] = info[0, 12:24]
    before = obs.clone()
    deploy.deploy_obs(env, table, 8, obs)
    assert torch.equal(obs, before)
    env.close()


def test_argument_errors():
    import torch
    from paddlerobotics_b200 import _lib
    lib = _lib.load()
    env = _env(4, "f32")
    h, s = env.h, _stream()
    od = env.observation_dim
    tab = torch.zeros(3, 12, device="cuda")
    obs, act, pol = env.obs, torch.zeros(4, 12, device="cuda"), torch.zeros(4, 12, device="cuda")
    rec = torch.zeros(2, od, device="cuda")
    p = lambda t: t.data_ptr()
    for args in ((None, 3, od - 12, 1, p(obs), None, 0), (p(tab), 3, od - 12, 1, None, None, 0), (p(tab), 0, od - 12, 1, p(obs), None, 0),
                 (p(tab), 3, -2, 1, p(obs), None, 0), (p(tab), 3, od - 11, 1, p(obs), None, 0), (p(tab), 3, od - 12, 1, p(obs), p(rec), 0)):
        assert lib.b2q_deploy_obs(h, *args, s) == -1, args
        assert b"b2q_deploy_obs" in lib.b2q_last_error(h)
    assert lib.b2q_deploy_obs(None, p(tab), 3, od - 12, 1, p(obs), None, 0, s) == -1
    for args in ((None, 0.3, p(tab), 3, p(act), None, 0), (p(pol), 0.3, None, 3, p(act), None, 0), (p(pol), 0.3, p(tab), 3, None, None, 0),
                 (p(pol), 0.3, p(tab), 0, p(act), None, 0), (p(pol), 0.3, p(tab), 3, p(act), p(rec), 0)):
        assert lib.b2q_deploy_act(h, *args, s) == -1, args
        assert b"b2q_deploy_act" in lib.b2q_last_error(h)
    assert lib.b2q_deploy_act(None, p(pol), 0.3, p(tab), 3, p(act), None, 0, s) == -1
    assert lib.b2q_deploy_obs(h, p(tab), 3, -1, 1, p(obs), p(rec), 2, s) == 0          # the accepted edges
    assert lib.b2q_deploy_obs(h, p(tab), 3, 0, 0, p(obs), None, 0, s) == 0
    torch.cuda.synchronize()
    env.close()


def test_graph_replay_advances_the_rows():
    """One iteration (obs kernel, student, act kernel, step) captured in a CUDA graph and replayed 6 times equals 6 eager iterations bit
    for bit, records included: the rows advance with the device step counters."""
    import torch
    from paddlerobotics_b200 import deploy, deploy_test
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    cfg = deploy.deploy_config(deploy_test.parser().parse_args([]))
    student = MujocoAgent(46, 12); student.restore(STUDENT)
    table = np.load(CPG)
    _, xo = deploy_test.batch_layout(1, 10)
    runs = []
    for graphed in (False, True):
        env = VecQuadrupedalEnv(10, **cfg)
        tab = torch.as_tensor(table, dtype=env.dtype, device="cuda")
        rec_o, rec_a = torch.zeros(8, 46, device="cuda"), torch.zeros(8, 12, device="cuda")
        action = torch.zeros(10, 12, device="cuda")
        obs = env.reset(x_offset=xo)

        def iteration():
            deploy.deploy_obs(env, tab, len(table), obs, rec_o)
            deploy.deploy_act(env, student.predict_batch(obs), 0.3, tab, len(table), action, rec_a)
            env.step(action)
        if graphed:
            torch.cuda.synchronize()
            g, cap = torch.cuda.CUDAGraph(), torch.cuda.Stream()
            cap.wait_stream(torch.cuda.current_stream())
            with torch.cuda.graph(g, stream=cap):
                iteration()
            torch.cuda.current_stream().wait_stream(cap)
            for _ in range(6):
                g.replay()
        else:
            for _ in range(6):
                iteration()
        torch.cuda.synchronize()
        runs.append([t.cpu().numpy() for t in (env.obs, env.info, action, rec_o, rec_a)] + [_step_counts(env)])
        env.close()
    assert (runs[1][-1] == 6).all()
    for a, b in zip(*runs):
        assert np.array_equal(a, b)
    assert (runs[1][3][6:] == 0).all() and (runs[1][3][:6] != 0).any(axis=1).all()


class _Replay:
    """A 46-input student for rehearse that returns, on its i-th call, the policy output the shipped student gave the ETG-mode loop at
    step i, and keeps the observation and the previous step's joint angles it was called with."""

    obs_dim = 46

    def __init__(self, outs, env):
        self.outs, self.env, self.seen, self.q = outs, env, [], []

    def predict_batch(self, obs):                # obs is the float32 copy of a float64 handle's observation: keep the handle's own
        self.seen.append(self.env.obs.cpu().numpy()); self.q.append(self.env.info[:, 42:54].cpu().numpy())
        return self.outs[len(self.seen) - 1]


def test_control_law_matches_the_training_env_in_float64():
    """rehearse with a t0 = 0 table of the gait (w, b) against the shipped student driving the ETG-mode env with the in-kernel (w, b)
    (env.step(student(obs[:, 3:]) * 0.3)), on float64 stairstair handles over 100 steps at start offsets -0.1, -1/30 and +1/30: every env's observation
    (ETG-mode columns 3:) and joint angles at every step within 1e-8, with row i applied at step i and row i + 1 in the observation after it.

    The two laws differ by rounding only (NumPy's ETG table against the kernel's, and the order of pose + ETG + action): 6e-14 at step 1,
    growing to at most 2.2e-9 by step 100 (measured on H100).  rehearse is given the student's outputs of the ETG-mode loop, because the
    fused MLP rounds its input to bf16 and such a difference can flip one input's rounding.  The fourth env, at +0.1, is not bounded: there, at
    step 94, a 2.7e-11 difference crosses a discrete branch of the contact model and the gap jumps to 2.2e-4 (DESIGN §8f)."""
    from paddlerobotics_b200 import deploy, deploy_test, etg
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv, quadrupedal_config
    z = np.load(SHIPPED)
    w, b = z["w"], z["b"]
    student = MujocoAgent(46, 12); student.restore(STUDENT)
    _, xo = deploy_test.batch_layout(1, 4)
    steps = 100
    cfg_train, _ = quadrupedal_config(task="stairstair")
    tr = VecQuadrupedalEnv(4, precision="f64", **cfg_train)
    obs = tr.reset(w, b, x_offset=xo)
    tr_obs, tr_q, outs = [], [], []
    for _ in range(steps):
        tr_obs.append(obs[:, 3:].cpu().numpy())
        outs.append(student.predict_batch(obs[:, 3:].float()).clone())
        obs, _, _, info = tr.step(outs[-1].double() * 0.3)
        tr_q.append(info[:, 42:54].cpu().numpy())
    tr_obs.append(obs[:, 3:].cpu().numpy())
    dep = VecQuadrupedalEnv(4, precision="f64", **deploy.deploy_config(deploy_test.parser().parse_args([])))
    rp = _Replay(outs, dep)
    res = deploy.rehearse(dep, rp, etg.etg_act_table(w, b, steps + 1), steps, x_offset=xo)
    dep_obs = np.array(rp.seen + [dep.obs.cpu().numpy()])
    dep_q = np.array(rp.q[1:] + [dep.info[:, 42:54].cpu().numpy()])
    assert np.isfinite(dep_obs).all() and np.array_equal(res["obs"], dep_obs[:steps, 0])
    ok = slice(0, 3)                                             # x -0.1, -1/30, +1/30; env 3 (x +0.1) is printed, not bounded
    print("env 3 (x +0.1) obs gap:", np.abs(dep_obs - np.array(tr_obs))[:, 3].max())
    gaps = {"obs": np.abs(dep_obs - np.array(tr_obs))[:, ok].max(), "joint_angle": np.abs(dep_q - np.array(tr_q))[:, ok].max()}
    print("float64 gap of the table-driven law to the in-kernel ETG over %d steps:" % steps, gaps)
    for k, g in gaps.items():
        assert g <= 1e-8, (k, g)
    tr.close(); dep.close()


def _run(tmp_path, monkeypatch, argv, sub):
    from paddlerobotics_b200 import deploy_test
    d = tmp_path / sub
    d.mkdir()
    monkeypatch.chdir(d)
    recs, res = deploy_test.main(argv)
    return recs, res, np.load(d / "data" / "exp0_rpm.npz")


def test_shipped_pair_end_to_end(tmp_path, monkeypatch, capsys):
    """deploy_test with the shipped student and CPG stair table, --max_time 1: the .npz holds finite obs [100,46] and action [100,12], each
    recorded action is 0.3 * predict_batch(obs[i]) + table[i] bit for bit, two runs are identical, and the JSON line has every field."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent
    argv = ["--load", STUDENT, "--ETG_path", CPG, "--max_time", "1"]
    recs, res, z = _run(tmp_path, monkeypatch, argv, "a")
    lines = [json.loads(l) for l in capsys.readouterr().out.strip().splitlines()]
    assert lines == recs and len(recs) == 1
    assert set(recs[0]) == {"dynamic_param", "envs", "falls", "mean_length", "min_length", "mean_distance", "mean_velx", "success_rate"}
    assert recs[0]["dynamic_param"] == "nominal" and recs[0]["envs"] == 1
    print("shipped pair, nominal, x 0:", recs[0])
    obs, act = z["obs"], z["action"]
    assert obs.shape == (100, 46) and act.shape == (100, 12) and np.isfinite(obs).all() and np.isfinite(act).all()
    student = MujocoAgent(46, 12); student.restore(STUDENT)
    pol = student.predict_batch(torch.as_tensor(obs, dtype=torch.float32, device="cuda")).cpu().numpy()
    table = np.load(CPG)[:100].astype(np.float32)
    assert np.array_equal(act.astype(np.float32), np.float32(0.3) * pol + table)
    assert np.array_equal(obs[:, 34:].astype(np.float32), (table - ETG_MEAN.astype(np.float32)) * (1.0 / ETG_STD).astype(np.float32))
    recs2, _, z2 = _run(tmp_path, monkeypatch, argv, "b")
    assert recs2 == recs and np.array_equal(z2["obs"], obs) and np.array_equal(z2["action"], act)


def test_batch_bookkeeping(tmp_path, monkeypatch):
    """Two --dynamic_param groups, a drawn vector and the nominal dynamics planted beside it.  At --x_starts 3 each group's record is the
    NumPy reduction of rehearse's per-env results.  At --x_starts 8 each group fills one warp of the step kernel, and the planted nominal
    group equals a nominal-only run env for env, bit for bit.  (Groups that share a warp need not: when any robot of a warp needs
    joint-limit or knee rows, the whole warp runs the wider contact solve, whose rounding differs; DESIGN §8f.)"""
    p = str(tmp_path / "p.npy"); np.save(p, np.random.default_rng(3).uniform(-0.5, 0.5, 48))
    base = ["--load", STUDENT, "--ETG_path", CPG, "--max_time", "2"]
    recs, res, _ = _run(tmp_path, monkeypatch, base + ["--x_starts", "3", "--dynamic_param", p, "nominal"], "mixed3")
    assert [r["dynamic_param"] for r in recs] == [p, "nominal"]
    for g, r in enumerate(recs):
        m = slice(3 * g, 3 * g + 3)
        assert r == {"dynamic_param": r["dynamic_param"], "envs": 3, "falls": int(res["fall"][m].sum()), "mean_length": float(res["length"][m].mean()),
                     "min_length": int(res["length"][m].min()), "mean_distance": float(res["distance"][m].mean()),
                     "mean_velx": float(res["velx"][m].mean()), "success_rate": float(res["success"][m].mean())}
    print("mixed batch, x_starts 3:", recs)
    recs, res, _ = _run(tmp_path, monkeypatch, base + ["--x_starts", "8", "--dynamic_param", p, "nominal"], "mixed8")
    nrecs, nres, _ = _run(tmp_path, monkeypatch, base + ["--x_starts", "8"], "nominal8")
    assert nrecs == [recs[1]]
    for k in ("length", "fall", "distance", "velx", "success"):
        assert np.array_equal(res[k][8:], nres[k]), k
    for k in res["terms"]:
        assert np.array_equal(res["terms"][k][8:], nres["terms"][k]), k
    print("mixed batch, x_starts 8:", recs)
