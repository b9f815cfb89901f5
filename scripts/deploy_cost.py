"""Cost of one deployment-rehearsal control step (paddlerobotics_b200.deploy.rehearse) at 1 and at 4096 envs, with the two deployment kernels
(b2q_deploy_obs / b2q_deploy_act) and, alternated in the same run, with the same loop written in torch indexing and arithmetic.  Each
window is --steps control steps of obs -> student -> act -> env step -> episode statistics after a reset, timed with CUDA events; the
median and spread over --reps windows (after one warm-up) are printed per step.  The card's name, power limit and SM clocks are read in
the same run.

It also prints what the rehearsal of the shipped pair (the reference's StairStair3_BC1_itr_500383.pt student with its CPG stair table,
tests/golden) does on stairstair at nominal dynamics over --max_time seconds, per start offset, and the largest difference in the first
step's joint target between the engine's action filter (history started from the settled joint angles) and deployment's (started from the
default pose).

    python scripts/deploy_cost.py [--steps 200] [--reps 5] [--max_time 7] [--x_starts 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlerobotics_b200 import _lib, deploy, deploy_test  # noqa: E402
from paddlerobotics_b200.agent import MujocoAgent  # noqa: E402
from paddlerobotics_b200.env import VecQuadrupedalEnv  # noqa: E402
from paddlerobotics_b200.es import EpisodeStats  # noqa: E402

STUDENT = os.path.join(ROOT, "tests", "golden", "StairStair3_BC1_itr_500383.pt")
CPG = os.path.join(ROOT, "tests", "golden", "gait_action_list_CPG_stairstair7_12_3.npy")
POSE = np.array([0, 0.9, -1.8] * 4)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:     # the number is still reported, with the reason the card's limits are unknown
        return "nvidia-smi unavailable (%s)" % e


def step_costs(n, steps, reps, cfg, student, table):
    lib = _lib.load()
    env = VecQuadrupedalEnv(n, auto_reset=False, **cfg)
    dev, dt, stream = env.device, env.dtype, env._stream()
    rows = len(table)
    tab = torch.as_tensor(table, dtype=dt, device=dev)
    col = deploy.etg_col_of(env)
    mean = torch.tensor([2.1505982e-02, 3.6674485e-02, -6.0444288e-02, 2.4625482e-02, 1.5869144e-02, -3.2513142e-02, 2.1506395e-02,
                         3.1869926e-02, -6.0140789e-02, 2.4625063e-02, 1.1628972e-02, -3.2163858e-02], dtype=dt, device=dev)
    istd = 1.0 / torch.tensor([4.5967497e-02, 2.0340437e-01, 3.7410179e-01, 4.6187632e-02, 1.9441207e-01, 3.9488649e-01, 4.5966785e-02,
                               2.0323379e-01, 3.7382501e-01, 4.6188373e-02, 1.9457331e-01, 3.9302582e-01], dtype=torch.float64, device=dev).to(dt)
    stats = EpisodeStats(lib, n, dt, dev, deploy.TERMS)
    action = torch.empty(n, 12, dtype=dt, device=dev)
    rec_o, rec_a = torch.empty(steps, env.observation_dim, dtype=dt, device=dev), torch.empty(steps, 12, dtype=dt, device=dev)
    sc = torch.empty(n, dtype=torch.int32, device=dev)

    def kernels(obs, i):
        deploy.deploy_obs(env, tab, rows, obs, rec_o)
        deploy.deploy_act(env, student.predict_batch(obs), 0.3, tab, rows, action, rec_a)

    def torch_ops(obs, i):
        assert lib.b2q_get_step_count(env.h, sc.data_ptr(), stream) == 0
        r = tab.index_select(0, sc.long())
        obs[:, col:col + 12] = (r - mean) * istd
        rec_o[i] = obs[0]
        torch.add(student.predict_batch(obs) * 0.3, r, out=action)
        rec_a[i] = action[0]

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {"kernels": [], "torch": []}
    for rep in range(reps + 1):
        for name, law in (("kernels", kernels), ("torch", torch_ops)):
            obs = env.reset()
            stats.zero()
            torch.cuda.synchronize()
            e0.record()
            for i in range(steps):
                law(obs, i)
                obs, rew, done, info = env.step(action)
                stats.step(rew, done, info, stream)
            e1.record()
            torch.cuda.synchronize()
            if rep:
                out[name].append(e0.elapsed_time(e1) / steps)
    env.close()
    res = {"envs": n}
    for k, v in out.items():
        res["step_ms_" + k], res["step_ms_%s_spread" % k] = float(np.median(v)), [min(v), max(v)]
    return res


def filter_difference(student, table):
    """Largest |engine target - deployment target| over the 12 joints of the first step with --enable_action_filter 1."""
    from scipy import signal
    args = deploy_test.parser().parse_args(["--enable_action_filter", "1"])
    env = VecQuadrupedalEnv(1, precision="f64", **deploy.deploy_config(args))
    res = deploy.rehearse(env, student, table, 1)
    engine = env.info[0, 24:36].cpu().numpy()
    fs = 1.0 / deploy.CONTROL_DT
    b, a = signal.butter(2, 4.0 / (fs / 2.0))                    # action_filter.py: a 4 Hz 2nd-order Butterworth low-pass
    x = POSE + res["action"][0]
    dep = (b[0] * x + (b[1] + b[2]) * POSE - (a[1] + a[2]) * POSE) / a[0]      # init_history(default pose): EnvWrapper.py:311-313
    env.close()
    return float(np.abs(engine - dep).max())


def shipped_pair(max_time, x_starts):
    argv = ["--load", STUDENT, "--ETG_path", CPG, "--max_time", str(max_time), "--x_starts", str(x_starts), "--suffix", "deploy_cost"]
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:     # deploy_test writes data/{suffix}_rpm.npz under the working directory
        os.chdir(d)
        try:
            recs, res = deploy_test.main(argv)
        finally:
            os.chdir(cwd)
    _, xo = deploy_test.batch_layout(1, x_starts)
    per_env = [{"x0": float(x), "fall": bool(res["fall"][e]), "length": int(res["length"][e]), "distance_m": float(res["distance"][e])}
               for e, x in enumerate(xo)]
    return {"max_time": max_time, "steps": deploy_test.steps_of(deploy_test.parser().parse_args(argv)), "group": recs[0], "per_env": per_env}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200, help="control steps per timed window")
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--envs", type=int, nargs="+", default=[1, 4096])
    p.add_argument("--max_time", type=float, default=7)
    p.add_argument("--x_starts", type=int, default=5)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deploy_cost.py measures on the GPU: no CUDA device")
    cfg = deploy.deploy_config(deploy_test.parser().parse_args([]))
    student = MujocoAgent(46, 12)
    student.restore(STUDENT)
    table = np.load(CPG)
    name = torch.cuda.get_device_name(0)
    for n in args.envs:
        out = step_costs(n, args.steps, args.reps, cfg, student, table)
        out["device"], out["nvidia_smi"] = name, gpu_info()
        print(json.dumps(out), flush=True)
    print(json.dumps({"action_filter_first_target_max_abs_diff_rad": filter_difference(student, table)}), flush=True)
    print(json.dumps({"shipped_pair": shipped_pair(1, 1)}), flush=True)
    print(json.dumps({"shipped_pair": shipped_pair(args.max_time, args.x_starts), "device": name, "nvidia_smi": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
