"""What the per-episode training statistics and the evaluation block of train.py cost on this GPU (DESIGN §8):
    python scripts/train_stats_cost.py
1. b2q_train_episode_stats alone at 4096 and 65536 envs: 200 launches captured in one CUDA graph, timed with CUDA events over 20 replays.
2. train.main at 4096 envs on the captured iteration, with the statistics launch and with it replaced by a no-op, alternated, 5 runs each after
   one warm-up run of each: the median over runs of each run's median interval between log records, per control step.
3. One evaluation block (run_evaluate_episodes, deterministic actor, at most 601 steps) at --train_eval_envs 1 and 16.
The card, its power limit and SM clock are read in the same run."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from paddlerobotics_b200 import _lib, es, train
from paddlerobotics_b200.agent import MujocoAgent


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:            # the numbers stand without it, but say so
        return "unknown (%s)" % e


def kernel_alone(n, launches=200, replays=20):
    st = es.TrainEpisodeStats(_lib.load(), n, torch.device("cuda"), train.EVAL_TERMS)
    rew = torch.randn(n, device="cuda")
    info = torch.randn(n, 56, device="cuda")
    done = (torch.rand(n, device="cuda") < 0.01).to(torch.uint8)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for _ in range(launches):
            st.step(rew, done, info, stream)
    torch.cuda.current_stream().wait_stream(s)
    g.replay(); torch.cuda.synchronize()
    times = []
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); g.replay(); b.record(); b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / launches)
    return float(np.median(times)), float(np.min(times))


def iteration(with_stats, n=4096, iters=600):
    real = es.TrainEpisodeStats.step
    if not with_stats:
        es.TrainEpisodeStats.step = lambda self, *a: None
    try:
        log = train.main(["--num_envs", str(n), "--batch", "4096", "--warmup_steps", str(4 * n), "--log_every", "50", "--ES", "0",
                          "--max_steps", str(iters * n), "--task_mode", "stairstair"])
    finally:
        es.TrainEpisodeStats.step = real
    # records after the capture (iteration 5): the interval rate of each, as µs per control step
    per_step = [n / r["interval_env_steps_per_s"] * 1e6 for r in log if r["iters"] >= 100]
    return float(np.median(per_step))


def eval_block(k):
    args = train.parser().parse_args(["--train_eval_envs", str(k)])
    env = train.make_eval_env(args, train.train_env_config(args), k)
    agent = MujocoAgent(env.observation_dim, 12, seed=0)
    _, w, b = train.initial_etg(args)
    out = []
    for _ in range(3):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        r = train.run_evaluate_episodes(env, w, b, policy=lambda o, s: agent.predict_batch(o), act_bound=0.3, max_step=train.EVAL_MAX_STEP)
        torch.cuda.synchronize(); out.append((time.perf_counter() - t0, r["mean_length"]))
    env.close()
    return out


def main():
    res = {"card": card()}
    res["kernel_us"] = {n: kernel_alone(n) for n in (4096, 65536)}
    iteration(True); iteration(False)
    arms = {"with": [], "without": []}
    for _ in range(5):
        arms["with"].append(iteration(True))
        arms["without"].append(iteration(False))
    res["iteration_us"] = {k: {"median": float(np.median(v)), "runs": v} for k, v in arms.items()}
    res["eval_block_s"] = {k: eval_block(k) for k in (1, 16)}
    res["card_after"] = card()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
