"""What one --save_state write and one --resume read cost on this GPU (DESIGN §8g):
    python scripts/train_state_cost.py [--num_envs 4096] [--memory 1000000]
The training objects of train.py at the given size, with the replay memory full, are saved and restored once after one warm-up round
trip.  Each part (env, learner, replay, rest) is timed with CUDA events around its state_dict / load_state_dict, and a host clock times
the file write (write_atomic: torch.save, flush, fsync, rename) and the file read (torch.load).  The card's name and power limit are read
in the same run.  The state file goes to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from paddlerobotics_b200 import _lib, train
from paddlerobotics_b200.agent import MujocoAgent, SACLearner
from paddlerobotics_b200.es import SimpleGA, TrainEpisodeStats
from paddlerobotics_b200.replay import ReplayMemory


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:            # the numbers stand without it, but say so
        return "unknown (%s)" % e


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return out, e0.elapsed_time(e1) / 1e3, time.perf_counter() - t


def nbytes(x):
    if isinstance(x, torch.Tensor):
        return x.numel() * x.element_size()
    if isinstance(x, np.ndarray):
        return x.nbytes
    if isinstance(x, dict):
        return sum(nbytes(v) for v in x.values())
    if isinstance(x, (list, tuple)):
        return sum(nbytes(v) for v in x)
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--memory", type=int, default=1000000)
    a = ap.parse_args()
    args = train.parser().parse_args(["--num_envs", str(a.num_envs), "--memory", str(a.memory), "--ES", "0"])
    env, _ = train.make_envs(args, train.train_env_config(args))
    od = env.observation_dim
    learner = SACLearner(MujocoAgent(od, 12), args.batch)
    rpm = ReplayMemory(args.memory, od, 12, device_cursor=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for i in range(0, args.memory, a.num_envs):           # a full ring: the largest state a run writes
        k = min(a.num_envs, args.memory - i)
        rpm.append(torch.randn(k, od, generator=g, device="cuda"), torch.rand(k, 12, generator=g, device="cuda"), torch.randn(k, generator=g, device="cuda"),
                   torch.randn(k, od, generator=g, device="cuda"), torch.ones(k, device="cuda"))
    stats = TrainEpisodeStats(_lib.load(), a.num_envs, env.device, train.EVAL_TERMS)
    solver = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=40, param=np.zeros(12))
    obs = env.reset(*train.etg_prior()[1:3]).clone()
    parts = {"env": env, "learner": learner, "replay": rpm}
    path = os.path.join(tempfile.mkdtemp(), "state.pt")
    rec = {"card": card(), "num_envs": a.num_envs, "memory": a.memory, "obs_dim": od}
    for rnd in range(2):                                  # round 0 warms up every path
        save, state = {}, {}
        for k, o in parts.items():
            state[k], dev_s, host_s = timed(o.state_dict)
            save[k] = {"bytes": nbytes(state[k]), "event_s": dev_s}
        rest, dev_s, _ = timed(lambda: {"stats": stats.state_dict(), "solver": solver.state_dict(), "obs": obs.cpu(), "cuda_rng": torch.cuda.get_rng_state()})
        state.update(rest)
        save["rest"] = {"bytes": nbytes(rest), "event_s": dev_s}
        t = time.perf_counter(); train.write_atomic(path, state); save["file_write_s"] = time.perf_counter() - t
        save["file_bytes"] = os.path.getsize(path)
        load = {}
        t = time.perf_counter(); got = torch.load(path, map_location="cpu", weights_only=False); load["file_read_s"] = time.perf_counter() - t
        for k, o in parts.items():
            _, dev_s, _ = timed(lambda: o.load_state_dict(got[k]))
            load[k] = {"event_s": dev_s}
        _, dev_s, _ = timed(lambda: (stats.load_state_dict(got["stats"]), solver.load_state_dict(got["solver"]), obs.copy_(got["obs"]),
                                     torch.cuda.set_rng_state(got["cuda_rng"])))
        load["rest"] = {"event_s": dev_s}
        save["total_s"] = sum(v["event_s"] for v in save.values() if isinstance(v, dict)) + save["file_write_s"]
        load["total_s"] = sum(v["event_s"] for v in load.values() if isinstance(v, dict)) + load["file_read_s"]
        del got
    os.remove(path); os.rmdir(os.path.dirname(path))
    rec.update(save=save, resume=load)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
