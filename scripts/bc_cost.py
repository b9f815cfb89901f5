"""Cost of behaviour-cloning training (paddlerobotics_b200.bctrain), timed with CUDA events, median of several rounds with the compared
paths alternated inside one run.  Prints JSON lines and the card's name and power limit:

  * us per BC update at batch 1024: the eager SACLearner.bc_learn (host torch.randn for eps, parameter pull) against SACLearner.bc_sweep
    (device gather + counter-RNG update, G updates per CUDA graph) for several G;
  * the collection rate at 4096 envs in env-steps/s: BCReplayMemory.observe (one kernel) against obs2noise_batch + slice + append,
    each with the student's sample and the env step;
  * the projected wall time of BCtrain.py's default schedule (1e6 env steps, 10 passes per 1024 rows, batch 1024) from those numbers.

    python scripts/bc_cost.py [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paddlerobotics_b200 import bc  # noqa: E402
from paddlerobotics_b200.agent import MujocoAgent, SACLearner  # noqa: E402
from paddlerobotics_b200.bctrain import sweep_schedule  # noqa: E402
from paddlerobotics_b200.env import VecQuadrupedalEnv  # noqa: E402
from paddlerobotics_b200.etg import ETG_layer, Opt_with_points  # noqa: E402
from paddlerobotics_b200.terrain import make_terrain  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:     # the number is still reported, with the reason the card's limits are unknown
        return "nvidia-smi unavailable (%s)" % e


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3          # seconds


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--updates", type=int, default=512, help="BC updates per timed window")
    p.add_argument("--envs", type=int, default=4096)
    p.add_argument("--steps", type=int, default=50, help="control steps per timed collection window")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bc_cost.py measures on the GPU: no CUDA device")
    B, K, dev = 1024, args.updates, torch.device("cuda", 0)
    # ---- learner: a ring of random pairs (one permutation covers every timed window), a random expert
    rpm = bc.BCReplayMemory(K * B + B, 46, 49, device=dev)
    ref = torch.randn(rpm.max_size, 49, device=dev)
    rpm.ref_obs.copy_(ref); rpm.obs.copy_(ref[:, 3:]); rpm._size = rpm.max_size
    expert, student = MujocoAgent(49, 12, seed=1), MujocoAgent(46, 12, seed=2)
    L = SACLearner(student, B)
    perm = torch.randperm(rpm.max_size, device=dev)
    Gs = (8, 32, 128)

    def eager():
        for k in range(K):
            idx = perm[k * B:(k + 1) * B]
            L.bc_learn(*rpm.sample_batch_by_index(idx), expert)        # torch.randn eps + parameter pull per update, as MujocoAgent.BClearn
    sweeps = {G: (lambda G=G: L.bc_sweep(rpm, expert, perm, K, seed=3, graph_steps=G, pull=True)) for G in Gs}
    for f in [eager] + list(sweeps.values()):                          # warm-up: module load, tensor maps, graph capture
        f()
    t_upd = {"eager": []}
    t_upd.update({G: [] for G in Gs})
    for _ in range(args.rounds):
        t_upd["eager"].append(timed(eager) / K)
        for G, f in sweeps.items():
            t_upd[G].append(timed(f) / K)
    # ---- collection at `envs` envs on stairstair
    n = args.envs
    env = VecQuadrupedalEnv(n, auto_reset=True, max_episode_steps=401, heightfield=make_terrain("stairstair"), stuck_termination=1, body_collisions=1,
                            joint_limits=1, knee_contacts=1)
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    obs = env.reset(w, b).clone()
    ring = bc.BCReplayMemory(1 << 20, 46, 49, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    step = [0]

    def collect_fused():
        for _ in range(args.steps):
            a_obs = ring.observe(obs, step[0])
            act = L.actor.forward(a_obs, mode=1, seed=step[0] + 1)[0][0]
            obs.copy_(env.step(act * 0.3)[0]); step[0] += 1

    def collect_torch():
        for _ in range(args.steps):
            a_obs = bc.cal_agent_obs(obs, True, gen)
            ring.append(a_obs, obs)
            act = L.actor.forward(a_obs, mode=1, seed=step[0] + 1)[0][0]
            obs.copy_(env.step(act * 0.3)[0]); step[0] += 1
    for f in (collect_fused, collect_torch):
        f()
    t_col = {"observe": [], "obs2noise_batch+append": []}
    for _ in range(args.rounds):
        t_col["observe"].append(timed(collect_fused))
        t_col["obs2noise_batch+append"].append(timed(collect_torch))
    info, name = gpu_info(), torch.cuda.get_device_name(dev)
    med = {k: float(np.median(v)) for k, v in t_upd.items()}
    for k, v in t_upd.items():
        print(json.dumps({"bc_update": "eager bc_learn" if k == "eager" else "bc_sweep", "graph_steps": None if k == "eager" else k, "batch": B,
                          "us_per_update": med[k] * 1e6, "us_spread": [min(v) * 1e6, max(v) * 1e6], "device": name, "nvidia_smi": info}), flush=True)
    rate = {}
    for k, v in t_col.items():
        rate[k] = n * args.steps / float(np.median(v))
        print(json.dumps({"collection": k, "num_envs": n, "env_steps_per_s": rate[k], "spread": [n * args.steps / max(v), n * args.steps / min(v)],
                          "device": name, "nvidia_smi": info}), flush=True)
    # ---- BCtrain.py's default schedule: 1e6 env steps, TRAIN_PER_STEPS 1024, TRAIN_PER_TIME 10, BATCH 1024, memory 1e7, warm-up 200
    total_updates = sum(len(o) for it in range(int(1e6) // n + 1) for _, _, o, _ in sweep_schedule(it * n, n, 1024, 10, B, int(1e7), 200, 64))
    best = min(Gs, key=lambda G: med[G])
    print(json.dumps({"schedule": "BCtrain default (1e6 env steps)", "num_envs": n, "bc_updates": total_updates,
                      "collection_s": 1e6 / rate["observe"],
                      "projected_learner_s": {"eager bc_learn": total_updates * med["eager"], "bc_sweep G=%d" % best: total_updates * med[best]},
                      "device": name, "nvidia_smi": info}), flush=True)
    env.close()


if __name__ == "__main__":
    main()
