"""The DEVICE code of the step kernel (paddlerobotics_b200/csrc/b2q_sim.cuh), compiled for the CPU with the warp
shuffles replaced by a 4-thread lock-step exchange (tests/emu/), against the float64 oracle.  This is the CPU-side
check of the kernel logic; the `-m gpu` tests repeat it through the real C ABI on the H100."""
import sys
import os

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
from oracle import oracle as O  # noqa: E402


def _pair(precision, w, b, n=1, **kw):
    ocfg = O.default_config(**{k: v for k, v in kw.items() if k in ("action_interp", "torque_limit", "solver_iters", "action_repeat", "action_filter", "max_episode_steps", "clip_motor_commands", "max_angle_change")})
    e = emu.EmuEnv(n, precision, **kw)
    o = O.OracleEnv(ocfg)
    return e, o, e.reset(w, b), o.reset(w, b)


def test_f64_device_code_equals_oracle(etg_stable):
    """Independent formulations (composite-inertia/Schur + contact-space PGS vs link-coordinate ABA + DoF-space PGS)
    agree to rounding in float64: state, obs, reward, done, info, over 60 free-running steps."""
    w, b = etg_stable
    e, o, oe, oo = _pair(1, w, b)
    assert np.abs(e.get_state()[0] - o.get_state()).max() < 1e-10      # settled snapshot
    assert np.abs(oe[0] - oo).max() < 1e-9
    rng = np.random.default_rng(0)
    for k in range(60):
        a = rng.uniform(-0.2, 0.2, 12)
        ob, rw, dn, inf = o.step(a)
        ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(e.get_state()[0] - o.get_state()).max() < 1e-9, k
        assert np.abs(ob2[0] - ob).max() < 1e-8 and abs(rw2[0] - rw) < 1e-8 and bool(dn2[0]) == dn
        assert np.array_equal(ob2[0][3:7], ob[3:7])                    # contact flags bit-exact
        assert np.abs(inf2[0] - inf).max() < 1e-8
    e.close()


def test_f64_fall_reset_and_done_flags(etg_default):
    """Default (aggressive) ETG gait + large residuals: the robot falls; done/fall flags and the in-step auto reset
    (snapshot copy) agree with the oracle."""
    w, b = etg_default
    e = emu.EmuEnv(1, 1, auto_reset=1)
    o = O.OracleBatch(1, etg_w=w, etg_b=b)
    e.reset(w, b)
    rng = np.random.default_rng(3)
    ndone = 0
    for k in range(80):
        a = rng.uniform(-0.3, 0.3, (1, 12))
        ob, rw, dn, inf = o.step(a, auto_reset=True)
        ob2, rw2, dn2, inf2 = e.step(a)
        assert int(dn2[0]) == int(dn[0]), k
        assert np.abs(ob2[0] - ob[0]).max() < 1e-7, k
        assert abs(rw2[0] - rw[0]) < 1e-7
        ndone += int(dn[0])
    assert ndone >= 1
    e.close()


def test_f64_options_interp_torque_limit_latency(etg_stable):
    w, b = etg_stable
    # action interpolation (minitaur.py:1384-1401) + torque clip (laikago_motor.py:168-173)
    e, o, _, _ = _pair(1, w, b, action_interp=1, torque_limit=20.0)
    rng = np.random.default_rng(1)
    for k in range(15):
        a = rng.uniform(-0.3, 0.3, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(ob2[0] - ob).max() < 1e-8
    e.close()
    # Butterworth action filter (minitaur.py:250-251, action_filter.py:111-216) incl. history init at reset and auto-reset
    e, o, _, _ = _pair(1, w, b, action_filter=1)
    for k in range(15):
        a = rng.uniform(-0.3, 0.3, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(ob2[0] - ob).max() < 1e-8 and np.abs(inf2[0] - inf).max() < 1e-8, k
    e.reset(); o.reset()
    for k in range(5):
        a = rng.uniform(-0.3, 0.3, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(inf2[0] - inf).max() < 1e-8
    e.close()
    # A1._ClipMotorCommands (a1.py:428-458): target clipped to the current angle +-max_angle_change every substep; a large
    # residual makes the clip bind, and the clipped run must differ from the unclipped one
    e, o, _, _ = _pair(1, w, b, clip_motor_commands=1, max_angle_change=0.05)
    e0, _, _, _ = _pair(1, w, b)
    for k in range(12):
        a = rng.uniform(-0.6, 0.6, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a); ob0 = e0.step(a)[0]
        assert np.abs(ob2[0] - ob).max() < 1e-8 and np.abs(inf2[0] - inf).max() < 1e-8, k
    assert np.abs(ob2[0] - ob0[0]).max() > 1e-3
    e.close(); e0.close()
    # per-env episode truncation (per-env form of donef=(steps>max_step), train.py:147)
    e, o, _, _ = _pair(1, w, b, max_episode_steps=7)
    for k in range(9):
        a = rng.uniform(-0.1, 0.1, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert bool(dn2[0]) == dn == (k >= 6), k
    e.close()
    # control latency across control-step boundaries (minitaur.py:1172-1193): 0.0305 s = 15.25 substeps, ring depth 3
    p = O.default_param(); p[25] = 0.0305
    e = emu.EmuEnv(1, 1, ring_depth=3)
    e.set_dynamics(p[None, :]); e.reset(w, b)
    o = O.OracleEnv(O.default_config(), p); o.reset(w, b)
    for k in range(12):
        a = rng.uniform(-0.2, 0.2, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(ob2[0] - ob).max() < 1e-8, k
        assert abs(rw2[0] - rw) < 1e-8
    e.close()


def test_f64_randomised_dynamics_rows(etg_stable, golden):
    """Per-env dynamics (kp/kd, friction, masses, inertias, gravity) from the reference's param2dynamic_dict."""
    from paddlerobotics_b200.etg import param2dynamic_dict, dynamic_dict_to_row
    w, b = etg_stable
    rng = np.random.default_rng(5)
    rows = []
    for i in range(2):
        d = param2dynamic_dict(rng.uniform(-0.3, 0.3, 48))
        d["control_latency"] = 2.0 + 6 * i          # ms
        d["footfriction"] = 0.8
        rows.append(dynamic_dict_to_row(d))
    rows = np.array(rows)
    e = emu.EmuEnv(2, 1)
    e.set_dynamics(rows); e.reset(w, b)
    for i in range(2):
        o = O.OracleEnv(O.default_config(), rows[i]); o.reset(w, b)
        assert np.abs(e.get_state()[i] - o.get_state()).max() < 1e-9
    acts = rng.uniform(-0.1, 0.1, (5, 2, 12))
    outs = [e.step(a) for a in acts]
    for i in range(2):
        o = O.OracleEnv(O.default_config(), rows[i]); o.reset(w, b)
        for k in range(5):
            ob, rw, dn, inf = o.step(acts[k, i])
            assert np.abs(outs[k][0][i] - ob).max() < 1e-8
    e.close()


def test_f64_heightfield_terrain(etg_stable):
    w, b = etg_stable
    xs = -1.6 + 0.04 * np.arange(128)
    hf = 0.02 * np.sin(6 * xs)[None, :] * np.ones((128, 1)) + 0.01 * np.cos(5 * xs)[:, None]
    e = emu.EmuEnv(1, 1, heightfield=(hf, -1.6, -1.6, 0.04))
    cfg = O.default_config(); O.set_heightfield(cfg, hf, -1.6, -1.6, 0.04)
    o = O.OracleEnv(cfg)
    e.reset(w, b); o.reset(w, b)
    assert np.abs(e.get_state()[0] - o.get_state()).max() < 1e-9
    rng = np.random.default_rng(2)
    for k in range(25):
        a = rng.uniform(-0.1, 0.1, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(ob2[0] - ob).max() < 1e-8
    e.close()


def test_f32_device_code_drift_1000_steps(etg_stable):
    """float32 product arithmetic, free-running 400 steps on the stable gait: joint-state drift vs the f64 oracle
    stays <= 1e-4 rad (BASELINE.json tolerance), contact flags agree on >= 99% of steps."""
    w, b = etg_stable
    e, o, _, _ = _pair(0, w, b)
    rng = np.random.default_rng(0)
    worst_q, mism = 0.0, 0
    for k in range(400):
        a = rng.uniform(-0.1, 0.1, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a.astype(np.float32))
        worst_q = max(worst_q, np.abs(e.get_state()[0][13:25] - o.get_state()[13:25]).max())
        mism += int(not np.array_equal(ob2[0][3:7], ob[3:7]))
        assert not dn
    assert worst_q < 1e-4, worst_q
    assert mism <= 4
    e.close()


def test_f32_teacher_forced_step_error(etg_stable):
    """Teacher forcing (SURVEY §8d protocol 1): before every step the f64 oracle state is loaded into the f32 engine;
    one-step error <= 1e-4 relative on q, qd, pose; contact flags bit-exact."""
    w, b = etg_stable
    e, o, _, _ = _pair(0, w, b)
    rng = np.random.default_rng(7)
    for k in range(40):
        a = rng.uniform(-0.3, 0.3, 12)
        e.set_state(o.get_state()[None, :])
        # keep the contact warm start identical as well
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a.astype(np.float32))
        so, se = o.get_state(), e.get_state()[0]
        assert np.abs(se[13:25] - so[13:25]).max() < 1e-4 * max(1.0, np.abs(so[13:25]).max())
        assert np.abs(se[25:37] - so[25:37]).max() < 1e-4 * max(1.0, np.abs(so[25:37]).max()) + 2e-3
        assert np.abs(se[:7] - so[:7]).max() < 1e-4
    e.close()


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_f64_random_dynamics_terrain_latency(etg_stable, seed):
    """Randomised per-env dynamics rows (param2dynamic_dict, train.py:112-126: masses, inertias, gains, friction, gravity, latency),
    a random smooth height field and a control latency of several substeps: the device code in CPU emulation still equals the
    oracle to rounding over 25 free-running steps."""
    from paddlerobotics_b200.etg import param2dynamic_dict, dynamic_dict_to_row
    w, b = etg_stable
    rng = np.random.default_rng(seed)
    d = param2dynamic_dict(rng.uniform(-0.4, 0.4, 48)); d["control_latency"] = float(rng.uniform(1.0, 20.0)); d["footfriction"] = float(rng.uniform(0.5, 1.2))
    row = dynamic_dict_to_row(d)
    xs = -1.6 + 0.05 * np.arange(64)
    hf = 0.015 * np.sin(rng.uniform(3, 7) * xs)[None, :] * np.ones((64, 1)) + 0.01 * np.cos(rng.uniform(3, 7) * xs)[:, None]
    e = emu.EmuEnv(1, 1, ring_depth=3, heightfield=(hf, -1.6, -1.6, 0.05), action_interp=int(seed % 2))
    e.set_dynamics(row[None, :]); e.reset(w, b)
    cfg = O.default_config(action_interp=int(seed % 2)); O.set_heightfield(cfg, hf, -1.6, -1.6, 0.05)
    o = O.OracleEnv(cfg, row); o.reset(w, b)
    for k in range(25):
        a = rng.uniform(-0.2, 0.2, 12)
        ob, rw, dn, inf = o.step(a); ob2, rw2, dn2, inf2 = e.step(a)
        assert np.abs(ob2[0] - ob).max() < 1e-7 and abs(rw2[0] - rw) < 1e-7 and bool(dn2[0]) == dn, (seed, k)
    e.close()
