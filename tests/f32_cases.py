"""Shared pieces of the float32 teacher-forced parity tests: the per-feature cases, the teacher-forced comparison against the
float64 oracle, and the oracle's own sensitivity to f32-rounded inputs.  Used by tests/test_emu_f32.py (the device code in CPU
emulation) and tests/test_gpu_f32_parity.py (the product kernel on the GPU).

Teacher forcing: before every control step the oracle's 37-wide state is loaded into the float32 engine, both take the same action,
and the outputs are compared.  Errors are relative to max(1, |reference|_inf) per quantity; contact flags, done and the fall flag are
compared bit-exact.

The oracle's sensitivity on a step is how far the oracle's own outputs move when its input state and action are rounded to float32
(a clone of the oracle, stepped once).  The float32 engine cannot do better than that on a step, and where the dynamics are
ill-conditioned (a foot on a riser, a contact that switches on) it is large; a bound that is looser than 1e-4 is stated as a multiple
of it plus a floor."""
import ctypes as C

import numpy as np

from oracle import oracle as O

POSE = np.array([0.0, 0.9, -1.8] * 4)
OKEYS = {f[0] for f in O.Config._fields_}
MAKE_ENV_FEATS = dict(stuck_termination=1, body_collisions=1, joint_limits=1, knee_contacts=1)      # what make_env switches on
PRESETS = ("stairstair", "slopeslope", "stairslope", "slopestair", "terrain", "balancebeam")
NOISE = (0.01, 0.05, 0.1, 0.02, 0.04)
FALL, BADFOOT = 54, 6                                                                               # info columns: fall flag, badfoot term


def actions(kind, rng, k, n):
    """[n, 12] (or [n, 60] in HYBRID mode) actions of control step k."""
    if kind == "residual":
        return rng.uniform(-0.2, 0.2, (n, 12))
    if kind == "small":
        return rng.uniform(-0.05, 0.05, (n, 12))
    if kind == "torque":                                    # roughly the standing torques plus noise
        return np.array([0.0, 1.0, -6.0] * 4) + rng.uniform(-1, 1, (n, 12))
    if kind == "hybrid":                                    # per motor (q*, kp, qd*, kd, tau_ff)
        a = np.zeros((n, 12, 5)); a[:, :, 0] = POSE + rng.uniform(-0.2, 0.2, (n, 12)); a[:, :, 1] = rng.uniform(60, 140, (n, 12))
        a[:, :, 2] = rng.uniform(-1, 1, (n, 12)); a[:, :, 3] = rng.uniform(0.5, 3, (n, 12)); a[:, :, 4] = rng.uniform(-2, 2, (n, 12))
        return a.reshape(n, 60)
    if kind == "stops":                                     # knees and hips driven into their stops
        a = np.zeros((n, 12)); a[:, 2::3] = 1.2 * np.sin(0.3 * k); a[:, 0::3] = 0.9 * np.cos(0.25 * k)
        return a
    if kind == "knees":                                     # thigh 0.3, calf -2.6: the toes fold up and the robot comes down on its knees
        a = np.zeros((n, 12)); a[:, 1::3] = 0.3 - 0.9; a[:, 2::3] = -2.6 + 1.8
        return a
    raise ValueError(kind)


def latency_row(ms):
    from paddlerobotics_b200.etg import dynamic_dict_to_row
    return dynamic_dict_to_row({"control_latency": float(ms)})


# name -> (gait fixture, engine / oracle config, action kind, control steps, extras)
CASES = {
    "noise": ("stable", dict(noise_stdev=NOISE, noise_seed=99), "residual", 20, {}),
    "torque": ("stable", dict(motor_mode=1), "torque", 8, {}),
    "hybrid_filter": ("stable", dict(motor_mode=2, action_filter=1), "hybrid", 16, {}),
    "joint_limits": ("shipped", dict(joint_limits=1), "stops", 14, {}),
    "knee_jlim_body": ("default", dict(knee_contacts=1, joint_limits=1, body_collisions=1, etg_enabled=0), "knees", 24, dict(knee_rest=True)),
    "push_damping": ("stable", dict(external_force=1, base_damping=(0.04, 0.02, 0.04, 0.01)), "residual", 16, dict(force=(6.0, 25.0, -3.0))),
    "filter_interp_clip": ("stable", dict(action_filter=1, action_interp=1, clip_motor_commands=1, max_angle_change=0.15), "residual", 16, {}),
    "latency": ("stable", {}, "residual", 16, dict(latency_ms=12.0)),
    "layout_raw_units": ("stable", dict(sensor_motor=2, sensor_imu=2, obs_normal=0), "residual", 12, {}),
    "layout_subset": ("stable", dict(sensor_dis=0, sensor_contact=0, sensor_etg=0), "residual", 12, {}),
}
for _t in PRESETS:   # make_env's feature set on every terrain preset, the shipped gait started just before the obstacle
    CASES["make_env_" + _t] = ("shipped", dict(MAKE_ENV_FEATS, **(dict(etg_foot_y_inset=0.05) if _t == "balancebeam" else {})), "small", 30,
                               dict(task=_t, x_offset=0.55))


def case_inputs(name):
    """gait, config, action kind, steps, height field, dynamics row, x offset, push force and knee_rest (see `errors`) of a case."""
    gait, kw, kind, steps, extra = CASES[name]
    hf = None
    if "task" in extra:
        from paddlerobotics_b200.terrain import make_terrain
        hf = make_terrain(extra["task"])
    row = latency_row(extra["latency_ms"]) if "latency_ms" in extra else None
    return gait, kw, kind, steps, hf, row, extra.get("x_offset"), extra.get("force"), extra.get("knee_rest", False)


def make_oracle(kw, hf, w, b, row=None, x_offset=None, force=None, env_id=0):
    o = O.OracleEnv(oracle_config(kw, hf), row)
    o.e.env_id = env_id
    ob = o.reset(w, b, x_offset=0.0 if x_offset is None else x_offset)
    if force is not None:
        o.set_force(force)
    return o, ob


def sloped_field(edge_x, edge_y, n=40, cell=0.05):
    """An n x n sloped, gently rippled height field whose far x / y edges lie at edge_x / edge_y."""
    x0, y0 = edge_x - (n - 1) * cell, edge_y - (n - 1) * cell
    xs, ys = x0 + cell * np.arange(n), y0 + cell * np.arange(n)
    hf = 0.06 * (xs[None, :] - edge_x) + 0.04 * (ys[:, None] - edge_y) + 0.01 * np.sin(7 * xs)[None, :] * np.cos(5 * ys)[:, None]
    return hf, x0, y0, cell


# far-edge placements of the sloped field relative to the robot's toes at the reset pose (x 0.157 front / -0.198 hind, y +-0.13):
# every foot beyond the edge, the front / left feet on it, and the edge one cell past the outermost feet
EDGE_CASES = {
    "x_beyond": (-0.45, 0.9), "x_on": (0.157, 0.9), "x_inside": (0.207, 0.9),
    "y_beyond": (0.9, -0.35), "y_on": (0.9, 0.13), "y_inside": (0.9, 0.18),
    "corner_beyond": (-0.45, -0.35),
}


def oracle_config(kw, hf=None):
    c = O.default_config(**{k: v for k, v in kw.items() if k in OKEYS})
    if hf is not None:
        O.set_heightfield(c, *hf)
    return c


def flag_columns(kw):
    """obs columns that hold the contact flags (bit-exact), given the sensor layout switches."""
    if not kw.get("sensor_contact", 1):
        return np.arange(0)
    off = 3 if kw.get("sensor_dis", 1) else 0
    return np.arange(off, off + 4)


def clone(o, scratch=None):
    """A copy of an oracle env (all of its internal state: warm starts, filter and latency history, counters)."""
    c = scratch if scratch is not None else O.OracleEnv(o.cfg, settle=False)
    C.memmove(C.byref(c.e), C.byref(o.e), C.sizeof(O.Env))
    return c


def _rel(x, ref):
    x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
    if x.size == 0:
        return 0.0
    return float(np.abs(x - ref).max() / max(1.0, np.abs(ref).max()))


def errors(ob, rw, inf, st, oo, ro, io, so, flags, knee_rest=False, reward_p=5.0):
    """Relative errors of one step of one env: obs (without the flag columns), q-dot, reward, info (without the fall flag), and the
    absolute error of pose and joint angles.

    knee_rest: a knee sphere (radius 0.02 m) held up by the knee contact rows rests at 0.0200000 m, exactly on the 0.02 m threshold
    of the non-toe contact count (`badfoot`), so which side of it the knee lands on is decided by rounding and the count is
    ill-conditioned there.  The reward (which carries the term times reward_p) and info are then compared without the badfoot term, and
    the term separately (`badfoot`): it may differ only by whole contacts (w_badfoot = 0.1 each)."""
    keep = np.setdiff1d(np.arange(len(oo)), flags)
    ik = np.setdiff1d(np.arange(len(io)), [FALL] + ([BADFOOT] if knee_rest else []))
    bf = (inf[BADFOOT] - io[BADFOOT]) if knee_rest else 0.0
    return dict(obs=_rel(ob[keep], oo[keep]), qd=_rel(st[25:37], so[25:37]), rew=_rel([rw - reward_p * bf], [ro]), info=_rel(inf[ik], io[ik]),
                pose=float(np.abs(st[:25] - so[:25]).max()), badfoot=abs(bf / 0.1 - round(bf / 0.1)) if knee_rest else 0.0)


def exact_mismatch(ob, dn, inf, oo, do, io, flags):
    """None, or what differs among the bit-exact outputs (contact flags, done, fall flag)."""
    if not np.array_equal(np.asarray(ob)[flags], oo[flags]):
        return "contact flags %s vs %s" % (np.asarray(ob)[flags], oo[flags])
    if bool(dn) != bool(do):
        return "done %s vs %s" % (bool(dn), bool(do))
    if float(inf[FALL]) != io[FALL]:
        return "fall flag %s vs %s" % (inf[FALL], io[FALL])
    return None


def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def ulps(x, n=4):
    """x with every element moved by n float64 ulps (relative 2^-52 n), in a fixed alternating direction: the float64 counterpart of
    _f32 for the sensitivity of a float64 engine."""
    x = np.asarray(x, np.float64)
    sign = np.where(np.arange(x.size) % 2 == 0, 1.0, -1.0).reshape(x.shape)
    return x * (1.0 + sign * n * np.finfo(np.float64).eps)


_HIST_AT, _HIST_LEN = O.Env.hist.offset, O.Env.hist_head.offset + C.sizeof(C.c_int) - O.Env.hist.offset   # hist, hist_len, hist_head


def teacher_forced(eng, oracles, acts, flags, knee_rest=False, perturb=_f32):
    """Teacher-forced steps of an engine with n envs against n oracles.  `eng` has set_state([n,37]), get_state() -> [n,37] and
    step([n,A]) -> (obs, reward, done, info) as float64 numpy arrays.  Neither side resets: an env that falls goes on being compared
    (the knee contact rows only carry load once the robot is down).  Returns one record per (step, env):
    (k, i, errors, oracle sensitivity, mismatch or None).  The sensitivity is the oracle's response to `perturb` applied to its input
    state and action: float32 rounding by default, `ulps` for a float64 engine.

    Teacher forcing loads the state, not the observation history.  With a control latency longer than about one control step the
    delayed observation of step k reads substeps of step k - 1 (and k - 2), which the engine computed itself.  So the sensitivity clone
    carries its own history forward: from step 1 on it starts from the history its perturbed step left, and its response contains the
    previous steps' rounding as the engine's does.  Before that, the history is the settled snapshot's (see full_range.warmup_steps)."""
    scratch = [O.OracleEnv(o.cfg, settle=False) for o in oracles]
    hist = [None] * len(oracles)
    rec = []
    for k, a in enumerate(acts):
        eng.set_state(np.stack([o.get_state() for o in oracles]))
        pre = [clone(o, scratch[i]) for i, o in enumerate(oracles)]
        ob, rw, dn, inf = eng.step(a)
        st = eng.get_state()
        for i, o in enumerate(oracles):
            oo, ro, do, io = o.step(a[i])
            so = o.get_state()
            c = pre[i]
            if hist[i] is not None:
                C.memmove(C.addressof(c.e) + _HIST_AT, hist[i], _HIST_LEN)
            c.set_state(perturb(c.get_state()))
            sob, srw, _, sinf = c.step(perturb(a[i]))
            hist[i] = C.create_string_buffer(_HIST_LEN)
            C.memmove(hist[i], C.addressof(c.e) + _HIST_AT, _HIST_LEN)
            rec.append((k, i, errors(ob[i], rw[i], inf[i], st[i], oo, ro, io, so, flags, knee_rest, o.cfg.reward_p),
                        errors(sob, srw, sinf, c.get_state(), oo, ro, io, so, flags, knee_rest, o.cfg.reward_p),
                        exact_mismatch(ob[i], dn[i], inf[i], oo, do, io, flags)))
    return rec


METRICS = ("obs", "qd", "rew", "info", "badfoot")
FLOOR = 2.5e-5          # relative error any step may have whatever the oracle's sensitivity (about 4x the flat-ground median)


def worst(rec):
    """Largest relative error over obs / q-dot / reward / info, and the largest pose / joint-angle error, of a teacher-forced run."""
    return max(r[2][m] for r in rec for m in METRICS), max(r[2]["pose"] for r in rec)


def worst_excess(rec, floor):
    """Largest (kernel error - floor) / oracle sensitivity over the steps and the relative measures: the multiple of the oracle's own
    f32-input sensitivity that the kernel's error reaches above the floor."""
    return max((r[2][m] - floor) / max(r[3][m], 1e-300) for r in rec for m in METRICS)


def summary(name, rec):
    w, p = worst(rec)
    return "%-26s steps %3d  worst rel %.3g  pose %.3g  oracle f32-input sensitivity %.3g  excess over %.3g floor %.3g" % (
        name, len(rec), w, p, max(r[3][m] for r in rec for m in METRICS), FLOOR, worst_excess(rec, FLOOR))
