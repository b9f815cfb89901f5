"""Deployment rehearsal on the GPU — the batched counterpart of the reference's deployment/test.py (same flags and defaults, :108-126).

The student (`--load`, a 46-input BC checkpoint by default) and the exported `.npy` gait table (`--ETG_path`) drive simulated robots with
the deployment control law (deploy.py): int(max_time * 100) control steps of base + 0.3 * student(obs) + table[i], no sensor noise and no
episode logic.  Env 0's observations and actions go to data/{suffix}_rpm.npz as test.py:105 writes them; one JSON line per dynamics
group summarises what every env did (falls, lengths and distance, frozen at each env's first done).

Batch flags the reference does not have:
    --task_mode T               terrain (default stairstair)
    --dynamic_param P.npy ...   one env group per 48-vector (dynamic_train's dynamic_param{epoch}.npy); the word `nominal` is a group
                                with the nominal dynamics; no flag = one nominal group
    --x_starts K                K start offsets per group, evenly spaced in [-0.1, 0.1] m (the x_noise range), so the gait phase at the
                                first stair varies; 1 (default) = x 0
Env g * K + k is group g at offset k; env 0 is the first group at the first offset.  With K a multiple of 8 every group fills whole warps
of the step kernel and its results are bit for bit those of the group run alone; envs that share a warp with another group can differ
from that in the last bits (DESIGN §8f), which a fall on the stairs may amplify.

Not reproduced: the `input()` prompt, the wall-clock pacing with time.sleep, and the real-robot client (a1_robot over UDP): the rehearsal
runs the engine as fast as it goes.  --sensor_footpose is accepted and ignored, as test.py never passes it to the env.

    python -m paddlerobotics_b200.deploy_test --load student.pt --ETG_path gait.npy --max_time 5 --x_starts 8
"""
import argparse
import json
import os

import numpy as np
import torch

from .deploy import CONTROL_DT, deploy_config, obs_dim_of, rehearse
from .env import VecQuadrupedalEnv
from .etg import dynamic_dict_to_row, param2dynamic_dict

ACT_BOUND = 0.3             # test.py:67
X_RANGE = 0.1               # the x_noise range of env.reset (train.py:505)


def parser():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    # ---- test.py:108-126
    p.add_argument("--suffix", type=str, default="exp0")
    p.add_argument("--ETG_path", type=str, default="exp/stair_6_21/gait_action_list_ETG_stair.npy", help="the exported gait table (.npy [rows,12])")
    p.add_argument("--sensor_dis", type=int, default=0)
    p.add_argument("--sensor_motor", type=int, default=1)
    p.add_argument("--sensor_imu", type=int, default=1)
    p.add_argument("--sensor_contact", type=int, default=1)
    p.add_argument("--sensor_footpose", type=int, default=0, help="accepted and ignored (test.py never passes it to the env)")
    p.add_argument("--sensor_ETG", type=int, default=1)
    p.add_argument("--timesteps", type=int, default=5)
    p.add_argument("--timeinterval", type=int, default=1)
    p.add_argument("--RNN_mode", type=str, default="None")
    p.add_argument("--dt", type=float, default=0.026)
    p.add_argument("--max_time", type=float, default=1)
    p.add_argument("--normal", type=float, default=1)
    p.add_argument("--gait", type=int, default=0)
    p.add_argument("--load", type=str, default="", help="the student checkpoint (.pt)")
    p.add_argument("--enable_action_filter", type=int, default=0)
    # ---- batch
    p.add_argument("--task_mode", type=str, default="stairstair")
    p.add_argument("--dynamic_param", type=str, nargs="*", default=[], help="one env group per 48-vector .npy; `nominal` = nominal dynamics")
    p.add_argument("--x_starts", type=int, default=1, help="start offsets per group, evenly spaced in [-0.1, 0.1] m")
    return p


def steps_of(args):
    return int(args.max_time * 100)             # test.py:93


def check_args(args):
    """Everything the rehearsal refuses, before any device work.  Returns (table, student state dict)."""
    if args.gait:
        raise NotImplementedError("--gait %d: the Bezier gait wrapper is not provided" % args.gait)
    if args.RNN_mode not in ("None", "", None) and args.timesteps > 0:
        raise NotImplementedError("--RNN_mode %s with --timesteps %d: stacked or GRU observations are not provided" % (args.RNN_mode, args.timesteps))
    if abs(args.dt - CONTROL_DT) > 1e-12:
        raise ValueError("--dt %g: the engine's control step is %g s (13 substeps of 2 ms)" % (args.dt, CONTROL_DT))
    if args.x_starts < 1:
        raise ValueError("--x_starts %d: at least one start offset" % args.x_starts)
    steps = steps_of(args)
    if steps < 1:
        raise ValueError("--max_time %g: fewer than one control step" % args.max_time)
    if not args.load:
        raise ValueError("--load: a student checkpoint is required")
    for path in args.dynamic_param:
        if path != "nominal" and np.load(path).size != 48:
            raise ValueError("--dynamic_param %s: a 48-vector is required" % path)
    table = np.load(args.ETG_path)
    if table.ndim != 2 or table.shape[1] != 12:
        raise ValueError("--ETG_path %s: the gait table must be [rows, 12], got %s" % (args.ETG_path, table.shape))
    if table.shape[0] < steps + 1:
        raise ValueError("--ETG_path %s: %d rows, but --max_time %g runs %d steps and the last observation reads row %d"
                         % (args.ETG_path, table.shape[0], args.max_time, steps, steps))
    sd = torch.load(args.load, map_location="cpu")
    width = obs_dim_of(args.sensor_dis, args.sensor_motor, args.sensor_imu, args.sensor_contact, args.sensor_ETG)
    have = int(sd["actor_model.l1.weight"].shape[1])
    if have != width:
        raise ValueError("--load %s: the actor takes %d inputs, but the --sensor_* flags give a %d-wide observation" % (args.load, have, width))
    return table, sd


def batch_layout(groups, x_starts):
    """(group of each env [N], base x offset of each env [N]) for `groups` dynamics groups of x_starts offsets each: env g * K + k."""
    xs = np.linspace(-X_RANGE, X_RANGE, x_starts) if x_starts > 1 else np.zeros(1)
    return np.repeat(np.arange(groups), x_starts), np.tile(xs, groups)


def group_rows(paths):
    """[G,48] engine dynamics rows of the --dynamic_param list (`nominal` = the nominal row); labels."""
    if not paths:
        return dynamic_dict_to_row(None)[None], ["nominal"]
    rows = [dynamic_dict_to_row(None) if p == "nominal" else dynamic_dict_to_row(param2dynamic_dict(np.load(p).reshape(-1))) for p in paths]
    return np.stack(rows), list(paths)


def summarise(res, group, labels):
    """One record per dynamics group from rehearse's per-env results."""
    recs = []
    for g, label in enumerate(labels):
        m = group == g
        recs.append({"dynamic_param": label, "envs": int(m.sum()), "falls": int(res["fall"][m].sum()), "mean_length": float(res["length"][m].mean()),
                     "min_length": int(res["length"][m].min()), "mean_distance": float(res["distance"][m].mean()),
                     "mean_velx": float(res["velx"][m].mean()), "success_rate": float(res["success"][m].mean())})
    return recs


def main(argv=None):
    from .agent import MujocoAgent
    args = parser().parse_args(argv)
    table, sd = check_args(args)
    steps = steps_of(args)
    dyn, labels = group_rows(args.dynamic_param)
    group, xoff = batch_layout(len(labels), args.x_starts)
    env = VecQuadrupedalEnv(len(group), auto_reset=False, **deploy_config(args))
    if args.dynamic_param:
        env.set_dynamics(dyn[group])
    student = MujocoAgent(int(sd["actor_model.l1.weight"].shape[1]), 12)
    student.load_state_dict(sd)
    res = rehearse(env, student, table, steps, act_bound=ACT_BOUND, x_offset=xoff)
    env.close()
    os.makedirs("data", exist_ok=True)
    np.savez(os.path.join("data", args.suffix + "_rpm.npz"), action=res["action"], obs=res["obs"])      # test.py:105
    recs = summarise(res, group, labels)
    for r in recs:
        print(json.dumps(r), flush=True)
    return recs, res


if __name__ == "__main__":
    main()
