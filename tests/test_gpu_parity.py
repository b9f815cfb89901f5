"""Parity tests proper: the CUDA path, called through the C ABI (libb2q.so), against the float64 oracle on the same
seeded inputs.  Float tolerance as BASELINE.json states: <= 1e-4 on joint state and reward; contact flags bit-exact
(in teacher-forced and float64 modes)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch


def _np(t):
    return t.detach().double().cpu().numpy()


def test_config1_teacher_forced_1000_steps(torch_cuda, etg_default):
    """SURVEY §8d config 1 AS SPECIFIED, protocol (1): default gait Opt_with_points(0.1, 0.05), residual sequence
    default_rng(0).uniform(-1,1,(1000,12))*0.3, 1000 control steps including the falls and resets it produces; before every step the
    oracle state is loaded into the f32 engine.  Stated tolerance, no extra slack: <= 1e-4 on q and pose, <= 1e-4 relative on
    q-dot and reward (relative to max(1, |reference|_inf)); contact flags, done and fall bit-exact."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    env = VecQuadrupedalEnv(1, precision="f32")
    o = O.OracleEnv()
    env.reset(w, b); o.reset(w, b)
    acts = np.random.default_rng(0).uniform(-1, 1, (1000, 12)) * 0.3
    wq = wp = wqd = wr = 0.0
    resets = 0
    for k in range(1000):
        env.set_state(o.get_state()[None, :])
        ob, rw, dn, inf = env.step(acts[k][None, :].astype(np.float32))
        oo, ro, do, io = o.step(acts[k])
        st, so = _np(env.get_state())[0], o.get_state()
        wq = max(wq, np.abs(st[13:25] - so[13:25]).max()); wp = max(wp, np.abs(st[:7] - so[:7]).max())
        wqd = max(wqd, np.abs(st[25:37] - so[25:37]).max() / max(1.0, np.abs(so[25:37]).max()))
        wr = max(wr, abs(float(rw[0]) - ro) / max(1.0, abs(ro)))
        assert np.array_equal(_np(ob)[0][3:7], oo[3:7]), k
        assert bool(dn[0]) == do and float(inf[0, 54]) == io[54], k
        if do:
            o.reset(); env.reset(); resets += 1
    print("config-1 teacher-forced, 1000 steps, %d resets: q %.3g  pose %.3g  qd(rel) %.3g  reward(rel) %.3g" % (resets, wq, wp, wqd, wr))
    assert resets >= 10
    assert wq <= 1e-4 and wp <= 1e-4 and wqd <= 1e-4 and wr <= 1e-4, (wq, wp, wqd, wr)
    env.close()


def test_free_running_shipped_gait_1000_steps(torch_cuda, etg_shipped):
    """Protocol (2) on a gait that walks: W,b fitted from the reference's own gait_action_list_ETG_exp.npy (0.48 m/s open loop),
    1000 free-running control steps (13 000 substeps), product f32 kernel vs f64 oracle.  BASELINE target: joint-state drift
    <= 1e-4; the base travels ~12.6 m, its drift is asserted relative to that distance."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_shipped
    env = VecQuadrupedalEnv(1, precision="f32")
    o = O.OracleEnv()
    env.reset(w, b); o.reset(w, b)
    z = np.zeros((1, 12), np.float32)
    worst_q = worst_r = worst_p = 0.0
    mism = 0
    for k in range(1000):
        ob, rw, dn, inf = env.step(z)
        oo, ro, do, io = o.step(z[0])
        st, so = _np(env.get_state())[0], o.get_state()
        worst_q = max(worst_q, np.abs(st[13:25] - so[13:25]).max())
        worst_p = max(worst_p, np.abs(st[:3] - so[:3]).max())
        worst_r = max(worst_r, abs(float(rw[0]) - ro) / max(1.0, abs(ro)))
        mism += int(not np.array_equal(_np(ob)[0][3:7], oo[3:7]))
        assert not do and not bool(dn[0]), k
    dist = o.get_state()[0]
    print("f32 free-running 1000 steps on the shipped gait: q drift %.3g rad, base pos %.3g m over %.2f m, reward(rel) %.3g, contact-flag mismatches %d"
          % (worst_q, worst_p, dist, worst_r, mism))
    assert 0.3 * 26.0 < dist < 0.6 * 26.0
    assert worst_q <= 1e-4, worst_q
    assert worst_p <= 1e-4 * dist, (worst_p, dist)
    assert worst_r <= 1e-3
    assert mism <= 5
    env.close()


def test_physics_regression_shipped_gait_f32(torch_cuda, etg_shipped):
    """Pinned to reference-held data: the gait table the reference ships must WALK in this physics — forward speed in
    [0.3, 0.6] m/s, no fall in 600 control steps (the table's length), upright, on the product f32 kernel, for a whole batch."""
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_shipped
    env = VecQuadrupedalEnv(64, precision="f32")
    env.reset(w, b)
    x0 = env.get_state()[:, 0].clone()
    z = torch.zeros(64, 12, device="cuda")
    for k in range(600):
        ob, rw, dn, inf = env.step(z)
        assert int(dn.sum()) == 0, k
    st = env.get_state()
    v = (st[:, 0] - x0) / (600 * 0.026)
    assert ((v > 0.3) & (v < 0.6)).all(), v
    assert (st[:, 2] > 0.2).all() and (inf[:, 36:38].abs() < 0.3).all()      # base height, roll / pitch
    env.close()


def test_make_env_reference_default_constructor_on_stairs(torch_cuda, etg_shipped):
    """The reference's exact constructor line (ETGRL/train.py:305-309) with the DEFAULT flags of its argparse block (:455-505) —
    task_mode 'stairstair', POSITION mode, all sensors on, dynamic_param from param2dynamic_dict (40 ms control latency) — then 400
    control steps as run_train_episode does (reset(ETG_w, ETG_b, x_noise), step(action*act_bound, donef)).  And kernel == oracle on
    that terrain (f64)."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import make_env, SENSOR_MODE, Random_Param_Dict, VecQuadrupedalEnv
    from paddlerobotics_b200.etg import param2dynamic_dict, dynamic_dict_to_row
    from paddlerobotics_b200.terrain import make_terrain

    class MotorControlMode:       # stand-in for robot_config.MotorControlMode.POSITION (enum value 1)
        name, value = "POSITION", 1
    sensor_mode = dict(SENSOR_MODE); sensor_mode["RNN"] = {"time_steps": 5, "time_interval": 1, "mode": "None"}
    reward_param = dict(torso=1.5, feet=0.3, up=0.6, tau=0.07, stand=0, badfoot=0.1, footcontact=0.1)
    dynamic_param = param2dynamic_dict(np.zeros(48))
    env = make_env('Quadrupedal', task="stairstair", motor_control_mode=MotorControlMode, render=False, sensor_mode=sensor_mode,
                   normal=1, dynamic_param=dynamic_param, reward_param=reward_param,
                   ETG=1, ETG_T=0.5, reward_p=5, ETG_path="None", random_param=dict(Random_Param_Dict),
                   ETG_H=20, vel_d=0.5, step_y=0.05, enable_action_filter=0)
    assert env.observation_space.shape[0] == 49 and env.action_space.shape[0] == 12
    w, b = etg_shipped
    obs, info = env.reset(ETG_w=w, ETG_b=b, x_noise=0)
    rng = np.random.default_rng(0)
    steps, x = 0, 0.0
    for k in range(400):
        obs, r, d, info = env.step(rng.uniform(-1, 1, 12) * 0.05, donef=(k + 1 > 400))
        assert obs.shape == (49,) and np.isfinite(obs).all() and np.isfinite(r)
        steps += 1; x += info["velx"] * 0.026
        if d:
            obs, _ = env.reset(ETG_w=w, ETG_b=b, x_noise=0)
    assert steps == 400 and x > 0.3          # it walked towards the staircase (0.8 m ahead; foot friction is 0.2 in this dynamics row, the robot slips)
    env.close()
    # kernel == oracle on the same terrain and dynamics row (float64)
    hf = make_terrain("stairstair")
    row = dynamic_dict_to_row(dynamic_param)
    feats = dict(stuck_termination=1, body_collisions=1, joint_limits=1, knee_contacts=1)       # what make_env switches on
    cfg = O.default_config(**feats); O.set_heightfield(cfg, *hf)
    o = O.OracleEnv(cfg, row); v = VecQuadrupedalEnv(1, precision="f64", heightfield=hf, **feats)
    v.set_dynamics(row[None, :])
    assert np.abs(_np(v.reset(w, b, x_offset=[0.5]))[0] - o.reset(w, b, x_offset=0.5)).max() < 1e-9
    for k in range(60):
        a = rng.uniform(-0.05, 0.05, 12)
        ob, rw, dn, inf = v.step(a[None, :]); oo, ro, do, io = o.step(a)
        assert np.abs(_np(ob)[0] - oo).max() < 1e-7 and abs(float(rw[0]) - ro) < 1e-7 and bool(dn[0]) == do, k
    assert o.foot_world()[:, 2].max() > 0.06      # feet are on the stairs
    v.close()


def test_env_features_f64_equal_oracle(torch_cuda, etg_stable):
    """Round-2 features through the C ABI on the GPU (float64 build) == oracle: reduced sensor layout in raw units, sensor noise,
    TORQUE and HYBRID motor modes, base push + damping, x-offset reset."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    rng = np.random.default_rng(2)
    for kw, torque in ((dict(sensor_motor=2, sensor_imu=2, obs_normal=0, noise_stdev=(0.01, 0.05, 0.1, 0.02, 0.04), noise_seed=99), False),
                       (dict(motor_mode=1), True),
                       (dict(motor_mode=2), "hybrid"),
                       (dict(external_force=1, base_damping=(0.04, 0.02, 0.04, 0.01), body_collisions=1, stuck_termination=1), False),
                       (dict(joint_limits=1), False),
                       (dict(knee_contacts=1, joint_limits=1, body_collisions=1, etg_enabled=0), False)):
        n = 3
        env = VecQuadrupedalEnv(n, precision="f64", **kw)
        os_ = [O.OracleEnv(O.default_config(**kw)) for _ in range(n)]
        xo = np.array([0.0, 0.05, -0.03])
        ob0 = _np(env.reset(w, b, x_offset=xo))
        for i, o in enumerate(os_):
            o.e.env_id = i
            assert np.abs(ob0[i] - o.reset(w, b, x_offset=xo[i])).max() < 1e-9
        if kw.get("external_force"):
            f = rng.uniform(-20, 20, (n, 3)); env.set_external_force(f)
            for i, o in enumerate(os_):
                o.set_force(f[i])
        for k in range(8 if torque is True else 20):     # open-loop torques diverge exponentially: compare before the rounding differences are amplified
            a = (np.array([0.0, 1.0, -6.0] * 4) + rng.uniform(-1, 1, (n, 12))) if torque is True else rng.uniform(-0.2, 0.2, (n, 12))
            if torque == "hybrid":                  # per motor (q*, kp, qd*, kd, tau_ff): laikago_motor.py:152-164
                a5 = np.zeros((n, 12, 5)); a5[:, :, 0] = np.array([0.0, 0.9, -1.8] * 4) + a; a5[:, :, 1] = rng.uniform(60, 140, (n, 12)); a5[:, :, 2] = rng.uniform(-1, 1, (n, 12))
                a5[:, :, 3] = rng.uniform(0.5, 3, (n, 12)); a5[:, :, 4] = rng.uniform(-2, 2, (n, 12)); a = a5.reshape(n, 60)
            if kw.get("knee_contacts"):            # thigh 0.3, calf -2.6: the toes fold up and the robot comes down on its knee spheres
                a = a * 0; a[:, 1::3] = 0.3 - 0.9; a[:, 2::3] = -2.6 + 1.8
            elif kw.get("joint_limits"):           # drive the knees and hips into their stops (a1.py:186-223)
                a = a * 0; a[:, 2::3] = 1.2 * np.sin(0.3 * k); a[:, 0::3] = 0.9 * np.cos(0.25 * k)
            ob, rw, dn, inf = env.step(a)
            for i, o in enumerate(os_):
                oo, ro, do, io = o.step(a[i])
                assert _np(ob).shape[1] == oo.shape[0] == env.observation_dim
                tol = 1e-6 if torque is True else 1e-7        # open-loop torques: no PD loop damps the rounding differences of the two formulations
                assert np.abs(_np(ob)[i] - oo).max() < tol and abs(float(rw[i]) - ro) < tol and bool(dn[i]) == do, (kw, k, i)
                assert np.abs(_np(inf)[i] - io).max() < tol
                if kw.get("joint_limits") and not kw.get("knee_contacts"):
                    q = o.get_state()[13:25]
                    assert q[2::3].min() > -2.69653369433 - 2e-3 and q[2::3].max() < -0.916297857297 + 2e-3 and np.abs(q[0::3]).max() < 0.802851455917 + 2e-3
                if do:
                    break
            else:
                continue
            break
        env.close()


@pytest.mark.parametrize("case", range(8))
def test_random_feature_combinations_f64_equal_oracle(torch_cuda, etg_stable, case):
    """Randomised interplay of the feature switches (sensor layout x noise x motor mode x limits / knee contacts x terrain x filter / interpolation /
    command clip x the reference's dynamics randomisation) through the C ABI on the GPU, float64 build, three envs per handle == oracle."""
    from conftest import draw_feature_combo
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    w, b = etg_stable
    rng = np.random.default_rng(2000 + case)
    kw, hf = draw_feature_combo(rng)
    n = 3
    okeys = {f[0] for f in O.Config._fields_}
    rows = np.stack([dynamic_dict_to_row(param2dynamic_dict(rng.uniform(-0.3, 0.3, 48))) for _ in range(n)])
    ekw = dict(kw)
    if hf is not None:
        ekw["heightfield"] = hf
    env = VecQuadrupedalEnv(n, precision="f64", **ekw)
    env.set_dynamics(rows)
    os_ = []
    for i in range(n):
        ocfg = O.default_config(**{k: v for k, v in kw.items() if k in okeys})
        if hf is not None:
            O.set_heightfield(ocfg, *hf)
        o = O.OracleEnv(ocfg, rows[i]); o.e.env_id = i
        os_.append(o)
    xo = rng.uniform(-0.1, 0.1, n)
    ob0 = _np(env.reset(w, b, x_offset=xo))
    for i, o in enumerate(os_):
        assert np.abs(ob0[i] - o.reset(w, b, x_offset=xo[i])).max() < 1e-8, (kw, i)
    if kw["external_force"]:
        f = rng.uniform(-15, 15, (n, 3)); env.set_external_force(f)
        for i, o in enumerate(os_):
            o.set_force(f[i])
    pose = np.array([0.0, 0.9, -1.8] * 4)
    alive = [True] * n
    for k in range(6):
        if kw["motor_mode"] == 2:
            a = np.zeros((n, 12, 5)); a[:, :, 0] = pose + rng.uniform(-0.2, 0.2, (n, 12)); a[:, :, 1] = rng.uniform(60, 140, (n, 12)); a[:, :, 2] = rng.uniform(-1, 1, (n, 12))
            a[:, :, 3] = rng.uniform(0.5, 3, (n, 12)); a[:, :, 4] = rng.uniform(-2, 2, (n, 12)); a = a.reshape(n, 60)
        elif kw["motor_mode"] == 1:
            a = np.array([0.0, 1.0, -6.0] * 4) + rng.uniform(-1, 1, (n, 12))
        else:
            a = rng.uniform(-0.3, 0.3, (n, 12))
        ob, rw, dn, inf = env.step(a)
        for i, o in enumerate(os_):
            if not alive[i]:
                continue
            oo, ro, do, io = o.step(a[i])
            assert np.abs(_np(ob)[i] - oo).max() < 1e-6 and abs(float(rw[i]) - ro) < 1e-6 and bool(dn[i]) == do, (kw, k, i)
            assert np.abs(_np(inf)[i] - io).max() < 1e-6, (kw, k, i)
            alive[i] = not do
    env.close()


def test_latency_beyond_the_ring_is_an_error(torch_cuda):
    """ADVICE r1: a control latency the observation ring cannot serve must be refused, not clamped."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import dynamic_dict_to_row
    env = VecQuadrupedalEnv(2, ring_depth=1)
    with pytest.raises(RuntimeError, match="ring_depth"):
        env.set_dynamics(np.stack([dynamic_dict_to_row({"control_latency": 40.0})] * 2))
    env.close()
    env = VecQuadrupedalEnv(2)                                                   # default ring depth 4 serves up to 100 ms
    env.set_dynamics(np.stack([dynamic_dict_to_row({"control_latency": 80.0})] * 2))
    env.close()


def test_f64_kernels_equal_oracle(torch_cuda, etg_stable):
    """float64 build of the same kernels == oracle to rounding (two independent formulations)."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    env = VecQuadrupedalEnv(3, precision="f64")
    o = [O.OracleEnv() for _ in range(3)]
    obs = _np(env.reset(w, b))
    for i in range(3):
        assert np.abs(obs[i] - o[i].reset(w, b)).max() < 1e-9
        assert np.abs(_np(env.get_state())[i] - o[i].get_state()).max() < 1e-10
    rng = np.random.default_rng(0)
    for k in range(100):
        a = rng.uniform(-0.2, 0.2, (3, 12))
        ob, rw, dn, inf = env.step(a)
        ob, rw, dn, inf, st = _np(ob), _np(rw), _np(dn), _np(inf), _np(env.get_state())
        for i in range(3):
            oo, ro, do, io = o[i].step(a[i])
            assert np.abs(st[i] - o[i].get_state()).max() < 1e-8, (k, i)
            assert np.abs(ob[i] - oo).max() < 1e-7 and abs(rw[i] - ro) < 1e-7 and bool(dn[i]) == do
            assert np.array_equal(ob[i][3:7], oo[3:7])
            assert np.abs(inf[i] - io).max() < 1e-7
    env.close()


def test_f32_free_running_1000_steps_drift(torch_cuda, etg_stable):
    """Config-1 style correctness run (1 env, flat plane, 1000 control steps, seeded residual sequence): product f32
    kernel vs f64 oracle, free running.  Joint state <= 1e-4, reward <= 1e-4 relative-ish, base pose drift reported."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    env = VecQuadrupedalEnv(1, precision="f32")
    o = O.OracleEnv()
    env.reset(w, b); o.reset(w, b)
    acts = np.random.default_rng(0).uniform(-1, 1, (1000, 12)) * 0.1
    worst_q = worst_r = worst_p = 0.0
    mism = 0
    for k in range(1000):
        ob, rw, dn, inf = env.step(acts[k][None, :].astype(np.float32))
        oo, ro, do, io = o.step(acts[k])
        st = _np(env.get_state())[0]
        worst_q = max(worst_q, np.abs(st[13:25] - o.get_state()[13:25]).max())
        worst_p = max(worst_p, np.abs(st[:3] - o.get_state()[:3]).max())
        worst_r = max(worst_r, abs(float(rw[0]) - ro))
        mism += int(not np.array_equal(_np(ob)[0][3:7], oo[3:7]))
        assert not do
    print("f32 1000-step drift: q %.3g rad, base pos %.3g m, reward %.3g, contact-flag mismatches %d/1000" % (worst_q, worst_p, worst_r, mism))
    # stable gait + +-0.1 residual noise: the noise makes the free-running comparison chaotic (CPU emulation of the same f32 code gives
    # 0.8e-4 .. 3.3e-4 depending on FMA contraction, DESIGN.md §6); the <=1e-4 target is asserted on the noise-free walking run above
    assert worst_q < 5e-4
    assert worst_r < 1e-2
    assert worst_p < 2e-3
    assert mism <= 10
    env.close()


def test_f32_teacher_forced(torch_cuda, etg_default):
    """Teacher forced on the aggressive default gait with +-0.3 residuals (BASELINE config 1 inputs), incl. falls."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    env = VecQuadrupedalEnv(1, precision="f32")
    o = O.OracleEnv()
    env.reset(w, b); o.reset(w, b)
    acts = np.random.default_rng(0).uniform(-1, 1, (60, 12)) * 0.3
    for k in range(60):
        env.set_state(o.get_state()[None, :])
        ob, rw, dn, inf = env.step(acts[k][None, :].astype(np.float32))
        oo, ro, do, io = o.step(acts[k])
        st, so = _np(env.get_state())[0], o.get_state()
        assert np.abs(st[13:25] - so[13:25]).max() < 1e-4
        assert np.abs(st[:7] - so[:7]).max() < 1e-4
        assert np.abs(st[25:37] - so[25:37]).max() <= 1e-4 * max(1.0, np.abs(so[25:37]).max())
        assert abs(float(rw[0]) - ro) <= 1e-4 * max(1.0, abs(ro))
        assert np.array_equal(_np(ob)[0][3:7], oo[3:7])
        assert bool(dn[0]) == do
        if do:
            o.reset(); env.reset()
    env.close()


def test_batch_4096_properties(torch_cuda, etg_default):
    """Full-size batch (BASELINE configs[1]): size-independent properties — identical envs given identical inputs stay
    bit-identical (determinism across warps/CTAs), envs are independent, auto-reset works, outputs finite."""
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    n = 4096
    env = VecQuadrupedalEnv(n, auto_reset=True)
    obs0 = env.reset(w, b).clone()
    assert torch.equal(obs0, obs0[0:1].expand_as(obs0))
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    half = torch.rand(n // 2, 12, device="cuda", generator=g) * 0.6 - 0.3
    ndone = 0
    for k in range(120):
        a = torch.cat([half, half]) if k % 2 == 0 else torch.cat([half.flip(0), half.flip(0)])
        ob, rw, dn, inf = env.step(a)
        assert torch.equal(ob[: n // 2], ob[n // 2:]) and torch.equal(rw[: n // 2], rw[n // 2:]) and torch.equal(dn[: n // 2], dn[n // 2:])
        assert torch.isfinite(ob).all() and torch.isfinite(rw).all()
        ndone += int(dn.sum())
    assert ndone > 0                                   # falls happened and were auto-reset
    st = env.get_state()
    assert torch.isfinite(st).all() and (st[:, 2] > 0.05).all()
    env.close()


def test_randomised_dynamics_latency_terrain_f64(torch_cuda, etg_stable):
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import param2dynamic_dict, dynamic_dict_to_row
    w, b = etg_stable
    rng = np.random.default_rng(5)
    rows = []
    for i in range(4):
        d = param2dynamic_dict(rng.uniform(-0.3, 0.3, 48)); d["control_latency"] = 2.0 + 9.5 * i; d["footfriction"] = 0.8
        rows.append(dynamic_dict_to_row(d))
    rows = np.array(rows)
    xs = -1.6 + 0.04 * np.arange(128)
    hf = 0.02 * np.sin(6 * xs)[None, :] * np.ones((128, 1)) + 0.01 * np.cos(5 * xs)[:, None]
    env = VecQuadrupedalEnv(4, precision="f64", ring_depth=4, heightfield=(hf, -1.6, -1.6, 0.04), action_interp=1, action_filter=1,
                            clip_motor_commands=1, max_angle_change=0.15)
    env.set_dynamics(rows); env.reset(w, b)
    cfg = O.default_config(action_interp=1, action_filter=1, clip_motor_commands=1, max_angle_change=0.15); O.set_heightfield(cfg, hf, -1.6, -1.6, 0.04)
    os_ = [O.OracleEnv(cfg, rows[i]) for i in range(4)]
    for o in os_:
        o.reset(w, b)
    for k in range(40):
        a = rng.uniform(-0.15, 0.15, (4, 12))
        ob, rw, dn, inf = env.step(a)
        for i in range(4):
            oo, ro, do, io = os_[i].step(a[i])
            assert np.abs(_np(ob)[i] - oo).max() < 1e-7, (k, i)
            assert abs(float(rw[i]) - ro) < 1e-7
    env.close()


def test_make_env_reference_call_shapes(torch_cuda, etg_default):
    """The reference's N=1 call surface (train.py:131,147; env_test.py:43-58): info['ETG_act'] over zero-residual steps
    reproduces the golden-table convention sample k = ETG(0.026*(k+1))."""
    from paddlerobotics_b200.env import make_env
    from paddlerobotics_b200.etg import etg_act_table
    w, b = etg_default
    env = make_env("Quadrupedal", task="ground", render=False, ETG=1, ETG_T=0.5, reward_p=5, vel_d=0.5, stuck_termination=0)
    assert env.observation_space.shape[0] == 49 and env.action_space.shape[0] == 12
    obs, info = env.reset(ETG_w=w, ETG_b=b, x_noise=0)
    assert obs.shape == (49,)
    tab = etg_act_table(w, b, 10, t0=0.026)
    for k in range(10):
        obs, r, d, info = env.step(np.zeros(12), donef=False)
        assert isinstance(r, float) and isinstance(d, bool) and {"velx", "ETG_act", "joint_angle", "obs-IMU", "real_action", "torso", "tau"} <= set(info)
        assert np.abs(info["ETG_act"] - tab[k]).max() < 2e-6
    obs, r, d, info = env.step(np.zeros(12), donef=True)
    assert d is True


def test_es_population_fitness_vs_oracle(torch_cuda, golden):
    """a15: population of ETG individuals (SimpleGA.ask -> Opt_with_points), each rolled out `rollouts` times on the
    GPU with first-done freezing; fitness vector == serial oracle evaluation (train.py:404-413 semantics)."""
    import torch
    from oracle import oracle as O
    from paddlerobotics_b200.es import PopulationEvaluator, SimpleGA, solutions_to_etg
    np.random.seed(0)
    ga = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.25, weight_decay=0.005, popsize=4, param=np.zeros(12))
    sol = ga.ask()
    w, b = solutions_to_etg(sol, golden["opt_points"], golden["opt_w0"], golden["opt_b0"])
    pop, rollouts, T = 4, 2, 45
    ev = PopulationEvaluator(pop, rollouts, max_steps=T, precision="f64")
    noise = np.random.default_rng(0).uniform(-0.3, 0.3, (T, pop * rollouts, 12))
    fit, mlen = ev.evaluate(w, b, residual_noise=torch.tensor(noise, device="cuda"))
    ref_fit, ref_len = np.zeros(pop), np.zeros(pop)
    for i in range(pop):
        for r in range(rollouts):
            o = O.OracleEnv(); o.reset(w[i], b[i])
            for k in range(T):
                _, rew, done, _ = o.step(noise[k, i * rollouts + r])
                ref_fit[i] += rew / rollouts; ref_len[i] += 1.0 / rollouts
                if done:
                    break
    assert np.abs(_np(fit) - ref_fit).max() < 1e-6, (_np(fit), ref_fit)
    assert np.array_equal(_np(mlen), ref_len)
    assert (ref_len < T).any()            # some episodes ended early (falls) and were frozen
    ga.tell(_np(fit))
    ev.env.close()


def test_host_buffer_api_equals_device_api(torch_cuda, etg_default):
    """b2q_step_host (numpy in/out through pinned buffers, the reference-facing call) == b2q_step on device tensors."""
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    a = VecQuadrupedalEnv(256, auto_reset=True); c = VecQuadrupedalEnv(256, auto_reset=True)
    a.reset(w, b); c.reset(w, b)
    rng = np.random.default_rng(0)
    for k in range(40):
        act = rng.uniform(-0.3, 0.3, (256, 12)).astype(np.float32)
        o1, r1, d1, _ = a.step(torch.tensor(act, device="cuda"))
        o2, r2, d2 = c.step_host(act)
        assert np.array_equal(o1.cpu().numpy(), o2) and np.array_equal(r1.cpu().numpy(), r2) and np.array_equal(d1.cpu().numpy(), d2)
    a.close(); c.close()


@pytest.mark.parametrize("n", [1, 13])
def test_ragged_batch_sizes_vs_oracle(torch_cuda, etg_stable, n):
    """Batch sizes that do not fill a warp (8 robots) — the masked lanes must neither store nor disturb the shuffles."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    env = VecQuadrupedalEnv(n, precision="f64")
    env.reset(w, b)
    os_ = [O.OracleEnv() for _ in range(n)]
    for o in os_:
        o.reset(w, b)
    rng = np.random.default_rng(n)
    for k in range(12):
        a = rng.uniform(-0.2, 0.2, (n, 12))
        ob, rw, dn, inf = env.step(a)
        for i in range(n):
            oo, ro, do, io = os_[i].step(a[i])
            assert np.abs(_np(ob)[i] - oo).max() < 1e-8 and abs(float(rw[i]) - ro) < 1e-8
    env.close()


def test_large_batch_and_error_paths(torch_cuda, etg_default):
    """65536 envs (16 x the benchmark batch): finite, duplicated envs identical; C ABI error codes instead of crashes."""
    import ctypes as C
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    env = VecQuadrupedalEnv(65536, auto_reset=True)
    env.reset(w, b)
    a = (torch.rand(8, 12, device="cuda") * 0.6 - 0.3).repeat(8192, 1)
    for k in range(10):
        ob, rw, dn, inf = env.step(a)
    assert torch.isfinite(ob).all() and torch.equal(ob[:8], ob[8:16]) and torch.equal(ob[:8], ob[-8:])
    lib = _lib.load()
    assert lib.b2q_step(env.h, None, 0, env.obs.data_ptr(), env.reward.data_ptr(), env.done.data_ptr(), env.info.data_ptr(), None) == -1
    assert b"null" in lib.b2q_last_error(env.h)
    assert lib.b2q_step(None, None, 0, None, None, None, None, None) == -1
    h = C.c_void_p()
    assert lib.b2q_sac_create(0, 49, 12, 100, 0.99, 0.005, 0.2, 3e-4, 3e-4, C.byref(h)) == -1      # batch not a multiple of 128
    assert lib.b2q_mlp_create(0, 80, 12, 1, C.byref(h)) == -1                                    # in_dim > 64
    env.close()


@pytest.mark.parametrize("n", [13, 64])
def test_step_host_io_modes_identical(torch_cuda, etg_stable, n, monkeypatch):
    """b2q_step_host: zero-copy pinned buffers (B2Q_HOST_IO=2, default), zero-copy actions only (1), memcpy staging (0) and
    PAGEABLE numpy buffers all return bit-identical obs / reward / done / info (the zero-copy info rows are their own store path);
    n=13 exercises the ragged last CTA."""
    import ctypes as C
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    rng = np.random.default_rng(7)
    acts = rng.uniform(-0.3, 0.3, (6, n, 12)).astype(np.float32)
    results = []
    for mode in ("2", "1", "0", "pageable"):
        monkeypatch.setenv("B2Q_HOST_IO", "2" if mode == "pageable" else mode)
        env = VecQuadrupedalEnv(n)
        env.reset(w, b)
        outs = []
        for a in acts:
            if mode == "pageable":
                o = np.empty((n, 49), np.float32); r = np.empty(n, np.float32); d = np.empty(n, np.uint8); inf = np.empty((n, 56), np.float32)
                rc = env.lib.b2q_step_host(env.h, a.ctypes.data_as(C.c_void_p), 0, o.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p),
                                           d.ctypes.data_as(C.c_void_p), inf.ctypes.data_as(C.c_void_p), None)
                assert rc == 0
            else:
                o, r, d, inf = env.step_host(a, info=True)
            outs.append((o.copy(), r.copy(), d.copy(), inf.copy()))
        results.append(outs)
        env.close()
    for other in results[1:]:
        for (o0, r0, d0, i0), (o1, r1, d1, i1) in zip(results[0], other):
            assert np.array_equal(o0, o1) and np.array_equal(r0, r1) and np.array_equal(d0, d1) and np.array_equal(i0, i1)
