"""The Bezier gait of deployment/test.py --gait 1 on the GPU: b2q_bezier_reset / b2q_bezier_act against the reference's trajectories
(tests/golden/bezier_gait.npz) and against the same arithmetic compiled for the CPU (bezier_host.py) on 4096 envs, the rehearsal's
applied joint targets rebuilt on the host, CUDA-graph replay, argument errors, and the deploy_bezier command end to end."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import bezier_host as H

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
STUDENT = os.path.join(GOLDEN, "StairStair3_BC1_itr_500383.pt")
POSE = np.array([0, 0.9, -1.8] * 4)


def _env(n, precision, **kw):
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    return VecQuadrupedalEnv(n, precision=precision, etg_enabled=0, **kw)


def _set_pose(env, q):
    """Each env's joint angles (b2q_get_state columns 13..24) set to q [N,12] after a reset; returns them in the handle's type."""
    import torch
    env.reset()
    s = env.get_state()
    s[:, 13:25] = torch.as_tensor(q, dtype=env.dtype, device=env.device)
    env.set_state(s)
    return s[:, 13:25].double().cpu().numpy()


def _drive(env, q, contact, rec_rows=0):
    """bezier_reset on poses q, then one bezier_act per step with the reference foot's bit contact[:, i] written into an observation of
    our own, on a zero action, and an env.step (which advances the step counters).  Returns the applied poses, the action increments
    [steps,N,12], the final gait state [N,18] and env 0's recorded feet."""
    import torch
    from paddlerobotics_b200 import deploy
    n, steps = contact.shape
    qa = _set_pose(env, q)
    state = torch.empty(n, deploy.BEZIER_STATE_DIM, dtype=torch.float64, device=env.device)
    deploy.bezier_reset(env, state)
    tb0 = state[:, :12].clone()
    obs = torch.zeros(n, env.observation_dim, dtype=env.dtype, device=env.device)
    col = deploy.contact_col_of(env)
    c = torch.as_tensor(contact, dtype=env.dtype, device=env.device)
    act = torch.zeros(steps, n, 12, dtype=env.dtype, device=env.device)
    zero = torch.zeros(n, 12, dtype=env.dtype, device=env.device)
    rec = torch.full((rec_rows, 4, 3), float("nan"), dtype=torch.float64, device=env.device) if rec_rows else None
    for i in range(steps):
        obs[:, col] = c[:, i]
        deploy.bezier_act(env, state, obs, act[i], rec)
        env.step(zero)
    torch.cuda.synchronize()
    return qa, tb0.cpu().numpy(), act.double().cpu().numpy(), state.cpu().numpy(), None if rec is None else rec.cpu().numpy()


def _close_with_nans(got, ref, tol):
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    err = float(np.abs(got[ok] - ref[ok]).max())
    assert err <= tol, err
    return err


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_against_the_reference_fixture(precision):
    """The 27 fixture cases as 27 envs.  float64: T_b0, env 0's recorded feet and every env's increment IK - POSE_ORI equal the
    reference within 1e-12, NaN where it has NaN.  float32: the handle holds its joint angles in float32, so the reference is the shared
    arithmetic (itself held to the fixture by test_bezier_cpu) on those angles; each increment is that float64 value rounded once."""
    g = dict(np.load(os.path.join(GOLDEN, "bezier_gait.npz")))
    env = _env(27, precision)
    qa, tb0, act, _, rec = _drive(env, g["q"], g["contact"], rec_rows=300)
    env.close()
    if precision == "f64":
        assert np.array_equal(qa, g["q"])
        feet, ang = g["feet"], g["ang"]
        assert np.abs(tb0.reshape(27, 4, 3) - g["tb0"]).max() <= 1e-12
    else:
        _, feet, ang, _ = H.rollout(qa, g["contact"])
    inc = ang.transpose(1, 0, 2) - POSE                                    # [steps, N, 12]
    print("feet of env 0: max |diff| %.3g" % _close_with_nans(rec, feet[0], 1e-12))
    if precision == "f64":
        print("increments: max |diff| %.3g" % _close_with_nans(act, inc, 1e-12))
    else:
        assert np.array_equal(np.isnan(act), np.isnan(inc))
        ok = ~np.isnan(inc)
        half_ulp = np.spacing(np.abs(inc[ok]).astype(np.float32)).astype(np.float64) / 2
        assert (np.abs(act[ok] - inc[ok]) <= half_ulp + 1e-12).all()          # round to nearest, once
        # where the float64 value is not within 1e-12 of a rounding midpoint the rounding is unambiguous, and the increment is exactly it
        # (near-zero abduction increments carry absolute errors ~1e-16, large next to their float32 ulp, and are left to the bound above)
        r = inc[ok].astype(np.float32).astype(np.float64)
        clear = np.abs(inc[ok] - r) < half_ulp - 1e-12
        print("float32 increments: %d of %d unambiguous roundings" % (clear.sum(), clear.size))
        assert clear.mean() > 0.5 and np.array_equal(act[ok][clear], r[clear])


def test_4096_envs_against_the_host_arithmetic():
    """4096 float64 envs, each with its own reset pose (some with nearly straight knees, so feet leave the reach) and its own contact
    stream: every env's increment at every one of 300 steps, and its final gait state, equal the CPU build of the same code within 1e-12."""
    rng = np.random.default_rng(3)
    n, steps = 4096, 300
    q = POSE + rng.uniform(-0.3, 0.3, (n, 12))
    q[::16] = np.array([0.05, 0.15, -0.3, -0.05, 0.1, -0.25, 0.08, 0.2, -0.35, -0.02, 0.05, -0.2]) + rng.uniform(-0.05, 0.05, (n // 16, 12))
    contact = (rng.random((n, steps)) < rng.uniform(0, 1, (n, 1))).astype(np.uint8)
    env = _env(n, "f64")
    qa, tb0, act, state, _ = _drive(env, q, contact)
    env.close()
    htb0, _, ang, flags = H.rollout(qa, contact)
    assert np.abs(tb0 - htb0.reshape(n, 12)).max() <= 1e-12
    err = _close_with_nans(act, ang.transpose(1, 0, 2) - POSE, 1e-12)
    print("4096 envs x %d steps: max |device - host| %.3g, %d NaN increments" % (steps, err, int(np.isnan(act).sum())))
    assert np.isnan(act).any()
    assert np.array_equal(state[:, 16], flags[:, -1, 0]) and np.array_equal(state[:, 17], flags[:, -1, 2])
    assert np.abs(state[:, 15] - flags[:, -1, 1]).max() <= 1e-12


@pytest.mark.parametrize("task", ["plane", "stairstair"])
def test_rehearsal_applies_ik_plus_student_plus_table(task):
    """rehearse(gait=True), 300 steps, the shipped student and a zero table: env 0's applied joint target at every step (info
    real_action) equals IK(feet_i) + 0.3 * student(obs_i) + table[i] rebuilt on the host from the recorded observation and feet, within
    float32 rounding; the recorded actions are the student plus the table, without the gait."""
    import torch
    from paddlerobotics_b200 import deploy, deploy_test
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    steps = 300
    student = MujocoAgent(46, 12); student.restore(STUDENT)
    env = VecQuadrupedalEnv(8, **deploy.deploy_config(deploy_test.parser().parse_args(["--task_mode", task])))
    targets = []
    step = env.step

    def recording_step(action):
        out = step(action)
        targets.append(out[3][0, 24:36].clone())
        return out
    env.step = recording_step
    table = np.zeros((steps + 1, 12))
    res = deploy.rehearse(env, student, table, steps, gait=True)
    env.close()
    tgt = torch.stack(targets).double().cpu().numpy()
    pol = student.predict_batch(torch.as_tensor(res["obs"], dtype=torch.float32, device="cuda")).double().cpu().numpy()
    assert np.array_equal(res["action"].astype(np.float32), np.float32(0.3) * pol.astype(np.float32) + table[:steps].astype(np.float32))
    host = H.ik(res["feet"]) + 0.3 * pol + table[:steps]
    live = res["length"][0]
    print("%s: env 0 ran %d steps, fell %s, distance %.3f m" % (task, live, bool(res["fall"][0]), res["distance"][0]))
    assert live >= 10 and np.isfinite(res["feet"]).all()
    err = _close_with_nans(tgt[:live], host[:live], 5e-6)
    print("applied target vs IK + 0.3 pi + table: max |diff| %.3g" % err)


def test_graph_replay_is_bit_identical():
    """One rehearsal iteration with the gait (obs kernel, student, act kernel, gait kernel, step) captured in a CUDA graph and replayed 12
    times equals 12 eager iterations bit for bit, gait state and feet record included: the gait reads each env's device step counter."""
    import torch
    from paddlerobotics_b200 import deploy, deploy_test
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    cfg = deploy.deploy_config(deploy_test.parser().parse_args([]))
    student = MujocoAgent(46, 12); student.restore(STUDENT)
    table = np.random.default_rng(5).uniform(-0.05, 0.05, (40, 12))
    _, xo = deploy_test.batch_layout(1, 16)
    runs = []
    for graphed in (False, True):
        env = VecQuadrupedalEnv(16, **cfg)
        tab = torch.as_tensor(table, dtype=env.dtype, device="cuda")
        gstate = torch.empty(16, deploy.BEZIER_STATE_DIM, dtype=torch.float64, device="cuda")
        rec_f = torch.zeros(14, 4, 3, dtype=torch.float64, device="cuda")
        action = torch.zeros(16, 12, device="cuda")
        obs = env.reset(x_offset=xo)
        deploy.bezier_reset(env, gstate)

        def iteration():
            deploy.deploy_obs(env, tab, len(table), obs)
            deploy.deploy_act(env, student.predict_batch(obs), 0.3, tab, len(table), action)
            deploy.bezier_act(env, gstate, obs, action, rec_f)
            env.step(action)
        if graphed:
            torch.cuda.synchronize()
            g, cap = torch.cuda.CUDAGraph(), torch.cuda.Stream()
            cap.wait_stream(torch.cuda.current_stream())
            with torch.cuda.graph(g, stream=cap):
                iteration()
            torch.cuda.current_stream().wait_stream(cap)
            for _ in range(12):
                g.replay()
        else:
            for _ in range(12):
                iteration()
        torch.cuda.synchronize()
        runs.append([t.cpu().numpy() for t in (env.obs, env.info, action, gstate, rec_f)])
        env.close()
    for a, b in zip(*runs):
        assert np.array_equal(a, b, equal_nan=True)
    assert (runs[1][4][12:] == 0).all() and np.isfinite(runs[1][4][:12]).all()
    assert (runs[1][3][:, 12] > 0).all()                                    # the gait clock runs after the five held steps


def test_argument_errors():
    import torch
    from paddlerobotics_b200 import _lib
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    env = _env(4, "f32")
    h, od = env.h, env.observation_dim
    st = torch.zeros(4, 18, dtype=torch.float64, device="cuda")
    act = torch.zeros(4, 12, device="cuda")
    rec = torch.zeros(2, 4, 3, dtype=torch.float64, device="cuda")
    p = lambda t: t.data_ptr()
    assert lib.b2q_bezier_reset(h, None, s) == -1 and b"b2q_bezier_reset" in lib.b2q_last_error(h)
    assert lib.b2q_bezier_reset(None, p(st), s) == -1
    for args in ((None, 0, p(env.obs), p(act), None, 0), (p(st), 0, None, p(act), None, 0), (p(st), 0, p(env.obs), None, None, 0),
                 (p(st), -1, p(env.obs), p(act), None, 0), (p(st), od, p(env.obs), p(act), None, 0), (p(st), 0, p(env.obs), p(act), p(rec), 0)):
        assert lib.b2q_bezier_act(h, *args, s) == -1, args
        assert b"b2q_bezier_act" in lib.b2q_last_error(h)
    assert lib.b2q_bezier_reset(h, p(st), s) == 0
    assert lib.b2q_bezier_act(h, p(st), od - 1, p(env.obs), p(act), p(rec), 2, s) == 0          # the accepted edges
    torch.cuda.synchronize()
    env.close()
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    etg = VecQuadrupedalEnv(4, etg_enabled=1)
    assert lib.b2q_bezier_reset(etg.h, p(st), s) == -1 and b"etg_enabled = 0" in lib.b2q_last_error(etg.h)
    assert lib.b2q_bezier_act(etg.h, p(st), 0, p(etg.obs), p(act), None, 0, s) == -1
    etg.close()


def test_deploy_bezier_end_to_end(tmp_path, monkeypatch, capsys):
    """deploy_bezier --gait 1 --max_time 3 --x_starts 8 with a zero table: it writes data/exp0_rpm.npz (obs [300,46], action [300,12] =
    0.3 * student, without the gait) and one JSON record marked "gait": 1."""
    zeros = str(tmp_path / "zeros.npy"); np.save(zeros, np.zeros((301, 12)))
    monkeypatch.chdir(tmp_path)
    from paddlerobotics_b200 import deploy_bezier
    recs, res = deploy_bezier.main(["--load", STUDENT, "--ETG_path", zeros, "--gait", "1", "--max_time", "3", "--x_starts", "8"])
    lines = [json.loads(l) for l in capsys.readouterr().out.strip().splitlines()]
    assert lines == recs and len(recs) == 1 and recs[0]["gait"] == 1 and recs[0]["envs"] == 8
    print("deploy_bezier --gait 1, zero table, 8 start offsets:", recs[0])
    z = np.load(tmp_path / "data" / "exp0_rpm.npz")
    assert z["obs"].shape == (300, 46) and z["action"].shape == (300, 12)
    assert res["feet"].shape == (300, 4, 3)
