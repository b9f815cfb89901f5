"""Deployment rehearsal: the control law of the reference's deployment/test.py:86-105 run by a batch of simulated robots.

Deployment does not run the in-kernel ETG generator.  Step i of an episode applies

    base + act_bound * student(obs) + table[i]                                    (test.py:93-99)

with the gait table exported as `.npy`, and the observation's ETG block is (table[iter] - ETG_mean) / ETG_std, iter = steps since reset
(EnvWrapper.py:103-107).  The env runs with ETG=0 (target = base pose + action); two kernels (include/b2q_deploy.h) write the ETG block
and the action from the table row each env's own step counter selects, so no argument changes from step to step.

Table phase: row k of a table made by etg.etg_act_table(w, b, rows) (t0 = 0) is ETG(0.026 k), the gait the training env applies at
step k, so that table reproduces the training env's control law.  `env_test --save 1` exports info["ETG_act"], whose row k is
ETG(0.026 (k + 1)): a student deployed with that table runs one control step ahead of the gait it was trained with (DESIGN §8f).

Bezier gait (test.py --gait 1, GaitWrapper of deployment/envs/EnvWrapper.py:123-193): the open-loop Bezier trot's joint angles take the
place of the base pose, so step i applies IK(feet_i) + act_bound * student(obs) + table[i].  Two more kernels (b2q_bezier_reset /
b2q_bezier_act, include/b2q_deploy.h) keep the gait's float64 state per env and add IK(feet_i) - POSE_ORI to the action (DESIGN §8f).
"""
import numpy as np
import torch

from . import _lib
from .env import _check, quadrupedal_config
from .es import EpisodeStats
from .train import EVAL_TERMS

CONTROL_DT = 0.026                              # test.py --dt default; the engine's control step (13 x 2 ms)
TERMS = EVAL_TERMS + ("velx", "fall")           # episode sums kept per env: the reward terms, Σ velx (distance) and the fall flag
BEZIER_STATE_DIM = 18                           # B2Q_BEZIER_STATE_DIM: float64 gait state per env (include/b2q_deploy.h)


def obs_dim_of(sensor_dis, sensor_motor, sensor_imu, sensor_contact, sensor_ETG):
    """The observation width the sensor flags select (test.py:26-46 get_obs_dim without the RNN stack)."""
    return ((24 if sensor_motor == 1 else 12 if sensor_motor == 2 else 0) + (3 if sensor_dis else 0) +
            (6 if sensor_imu == 1 else 3 if sensor_imu == 2 else 0) + (4 if sensor_contact else 0) + (12 if sensor_ETG else 0))


def deploy_config(args):
    """The env configuration of the rehearsal: quadrupedal_config's (joint limits, knee contacts, stuck termination and body
    collisions on, no sensor noise) with ETG=0, the sensor flags, `normal`, the action filter and the task's height field.
    VecQuadrupedalEnv keywords."""
    cfg, _ = quadrupedal_config(task=args.task_mode, normal=args.normal, ETG=0, enable_action_filter=args.enable_action_filter,
                                sensor_mode={"dis": args.sensor_dis, "motor": args.sensor_motor, "imu": args.sensor_imu,
                                             "contact": args.sensor_contact, "ETG": args.sensor_ETG})
    return cfg


def etg_col_of(env):
    """Column of the observation's ETG block (the last 12), or -1 when the sensor flags have none."""
    return env.observation_dim - 12 if env.cfg.sensor_etg else -1


def deploy_obs(env, table, rows, obs, rec_obs=None):
    """b2q_deploy_obs: the ETG block of obs [N,obs_dim] from table [rows,12] (device, the env's dtype) at each env's step counter."""
    p = lambda t: None if t is None else t.data_ptr()
    _check(env.lib, env.h, env.lib.b2q_deploy_obs(env.h, table.data_ptr(), rows, etg_col_of(env), int(env.cfg.obs_normal), obs.data_ptr(), p(rec_obs),
                                                  0 if rec_obs is None else rec_obs.shape[0], env._stream()), "b2q_deploy_obs")


def deploy_act(env, policy_out, act_bound, table, rows, action, rec_act=None):
    """b2q_deploy_act: action [N,12] = act_bound * policy_out (float32) + table row of each env's step counter."""
    p = lambda t: None if t is None else t.data_ptr()
    _check(env.lib, env.h, env.lib.b2q_deploy_act(env.h, policy_out.data_ptr(), float(act_bound), table.data_ptr(), rows, action.data_ptr(), p(rec_act),
                                                  0 if rec_act is None else rec_act.shape[0], env._stream()), "b2q_deploy_act")


def contact_col_of(env):
    """Column of the reference foot's FootContactSensor bit in the observation (the contact block follows BaseDisplacement)."""
    if not env.cfg.sensor_contact:
        raise ValueError("the Bezier gait reads the foot contacts: the observation has no FootContactSensor block (sensor_contact 0)")
    return 3 if env.cfg.sensor_dis else 0


def bezier_reset(env, state):
    """b2q_bezier_reset: state [N,BEZIER_STATE_DIM] float64 <- the feet of each env's current joint angles and a fresh gait clock."""
    _check(env.lib, env.h, env.lib.b2q_bezier_reset(env.h, state.data_ptr(), env._stream()), "b2q_bezier_reset")


def bezier_act(env, state, obs, action, rec_feet=None):
    """b2q_bezier_act: advances the gait of every env at its step counter, with the reference foot's contact bit from obs, and adds
    IK(feet) - POSE_ORI to action [N,12] in place; env 0's feet go to rec_feet [rows,4,3] float64 (or None)."""
    _check(env.lib, env.h, env.lib.b2q_bezier_act(env.h, state.data_ptr(), contact_col_of(env), obs.data_ptr(), action.data_ptr(),
                                                  None if rec_feet is None else rec_feet.data_ptr(), 0 if rec_feet is None else rec_feet.shape[0],
                                                  env._stream()), "b2q_bezier_act")


def rehearse(env, student, table, steps, act_bound=0.3, record=True, x_offset=None, gait=False):
    """One rollout of test.py's loop on every env of `env` (a VecQuadrupedalEnv built from deploy_config, no auto-reset): reset (base x
    offset x_offset [N] or None), then per step deploy_obs -> student.predict_batch -> deploy_act -> env.step -> EpisodeStats.step, and
    after the last step the observation test.py's last get_observation reads (table row `steps`).  No host sync until the end.
    With `gait` (test.py --gait 1) the Bezier gait runs too: bezier_reset after the reset and bezier_act between deploy_act and the step.

    Returns numpy per-env results, each frozen at the env's first done: length, fall (bool), distance (Σ velx * 0.026), velx (mean over
    the episode), success (fraction of steps with velx >= 0.3), terms {EVAL_TERMS name: episode sum}; with record, env 0's obs
    [steps,obs_dim] and action [steps,12] (test.py:97-98: the student plus the table, without the gait), and with the gait its feet
    [steps,4,3]."""
    table = np.asarray(table)
    if table.ndim != 2 or table.shape[1] != 12:
        raise ValueError("the gait table must be [rows, 12], got %s" % (table.shape,))
    if table.shape[0] < steps + 1:
        raise ValueError("the gait table has %d rows; %d steps read rows 0..%d" % (table.shape[0], steps, steps))
    if student.obs_dim != env.observation_dim:
        raise ValueError("the student takes %d inputs, the observation has %d columns" % (student.obs_dim, env.observation_dim))
    lib, n, dev, dt = _lib.load(), env.num_envs, env.device, env.dtype
    rows = int(table.shape[0])
    tab = torch.as_tensor(table, dtype=dt, device=dev).contiguous()
    rec_obs = torch.full((steps, env.observation_dim), float("nan"), dtype=dt, device=dev) if record else None
    rec_act = torch.full((steps, 12), float("nan"), dtype=dt, device=dev) if record else None
    stats = EpisodeStats(lib, n, dt, dev, TERMS)
    action = torch.empty(n, 12, dtype=dt, device=dev)
    stream = env._stream()
    if gait:
        gstate = torch.empty(n, BEZIER_STATE_DIM, dtype=torch.float64, device=dev)
        rec_feet = torch.full((steps, 4, 3), float("nan"), dtype=torch.float64, device=dev) if record else None
    obs = env.reset(x_offset=x_offset)
    if gait:
        bezier_reset(env, gstate)
    for _ in range(steps):
        deploy_obs(env, tab, rows, obs, rec_obs)
        pol = student.predict_batch(obs if dt == torch.float32 else obs.float())
        deploy_act(env, pol, act_bound, tab, rows, action, rec_act)
        if gait:
            bezier_act(env, gstate, obs, action, rec_feet)
        obs, rew, done, info = env.step(action)
        stats.step(rew, done, info, stream)
    deploy_obs(env, tab, rows, obs)
    length = stats.len.cpu().numpy()
    sums = stats.term_sum.double().cpu().numpy()
    col = {k: j for j, k in enumerate(TERMS)}
    out = {"length": length, "fall": sums[col["fall"]] > 0, "distance": sums[col["velx"]] * CONTROL_DT, "velx": sums[col["velx"]] / length,
           "success": stats.success_rate().double().cpu().numpy(), "terms": {k: sums[col[k]] for k in EVAL_TERMS}}
    if record:
        out["obs"], out["action"] = rec_obs.double().cpu().numpy(), rec_act.double().cpu().numpy()
        if gait:
            out["feet"] = rec_feet.cpu().numpy()
    return out
