"""Cost of the Bezier gait (deploy_bezier, test.py --gait 1) in a deployment-rehearsal control step at --envs envs: the same loop (obs kernel ->
student -> act kernel -> [gait kernel] -> env step -> episode statistics after a reset) with and without the gait, alternated in one run,
each window --steps control steps timed with CUDA events, median and spread over --reps windows after one warm-up.  The gait changes
how the robots move, and the step kernel's time depends on that (contact rows), so a third loop runs the gait kernel on a copy of the
action and discards it: its difference to the loop without the gait is the gait kernel's share of the step.  Then b2q_bezier_act
alone, --launches back-to-back launches between two events.  The card's name, power limit and SM clocks are read in the same run.

    python scripts/bezier_cost.py [--envs 4096] [--steps 200] [--reps 5] [--launches 2000]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, ROOT)
from deploy_cost import CPG, STUDENT, gpu_info  # noqa: E402
from paddlerobotics_b200 import _lib, deploy, deploy_test  # noqa: E402
from paddlerobotics_b200.agent import MujocoAgent  # noqa: E402
from paddlerobotics_b200.env import VecQuadrupedalEnv  # noqa: E402
from paddlerobotics_b200.es import EpisodeStats  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=200, help="control steps per timed window")
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--launches", type=int, default=2000)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bezier_cost.py measures on the GPU: no CUDA device")
    n, steps = args.envs, args.steps
    student = MujocoAgent(46, 12)
    student.restore(STUDENT)
    table = np.load(CPG)
    env = VecQuadrupedalEnv(n, auto_reset=False, **deploy.deploy_config(deploy_test.parser().parse_args([])))
    lib, dev, dt, stream = _lib.load(), env.device, env.dtype, env._stream()
    rows = len(table)
    tab = torch.as_tensor(table, dtype=dt, device=dev)
    stats = EpisodeStats(lib, n, dt, dev, deploy.TERMS)
    action = torch.empty(n, 12, dtype=dt, device=dev)
    gstate = torch.empty(n, deploy.BEZIER_STATE_DIM, dtype=torch.float64, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    scratch = torch.empty(n, 12, dtype=dt, device=dev)
    times = {"without_gait": [], "with_gait": [], "gait_discarded": []}
    for rep in range(args.reps + 1):
        for name in times:
            obs = env.reset()
            if name != "without_gait":
                deploy.bezier_reset(env, gstate)
            stats.zero()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                deploy.deploy_obs(env, tab, rows, obs)
                deploy.deploy_act(env, student.predict_batch(obs), 0.3, tab, rows, action)
                if name == "with_gait":
                    deploy.bezier_act(env, gstate, obs, action)
                elif name == "gait_discarded":          # the gait kernel's own cost: it runs, but the robots move as without it
                    scratch.copy_(action)
                    deploy.bezier_act(env, gstate, obs, scratch)
                obs, rew, done, info = env.step(action)
                stats.step(rew, done, info, stream)
            e1.record()
            torch.cuda.synchronize()
            if rep:
                times[name].append(e0.elapsed_time(e1) / steps)
    out = {"envs": n, "steps_per_window": steps, "reps": args.reps}
    for k, v in times.items():
        out["step_ms_" + k], out["step_ms_%s_spread" % k] = float(np.median(v)), [min(v), max(v)]
    # the gait kernel alone: the step counters stay put, so every launch advances the gait clock of a walking (timesteps > 5) env
    for _ in range(6):
        env.step(action)
    deploy.bezier_reset(env, gstate)
    for _ in range(20):
        deploy.bezier_act(env, gstate, env.obs, action)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.launches):
        deploy.bezier_act(env, gstate, env.obs, action)
    e1.record()
    torch.cuda.synchronize()
    out["bezier_act_us"] = e0.elapsed_time(e1) * 1000.0 / args.launches
    out["device"], out["nvidia_smi"] = torch.cuda.get_device_name(0), gpu_info()
    env.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
