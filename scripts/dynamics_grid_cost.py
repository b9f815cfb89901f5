"""What a dynamics-sweep evaluation costs on this GPU (DESIGN §8i):
    python scripts/dynamics_grid_cost.py [--repeats 3]
The wall time of whole --eval 1 --dynamics_grid 1 runs through the commands, set-up included (create, one set_dynamics with 82 settings'
rows and its settle, the episode of at most 601 steps, the records), host clock ending in a device synchronise:
1. pretrain with the shipped gait (the zero residual, which walks) on stairstair, --eval_envs 1 (82 envs) and 8 (656 envs);
2. train with a seeded actor and the shipped gait on stairstair, --eval_envs 8 (656 envs);
each beside the same command's plain --eval 1 at the same --eval_envs.  One untimed warm-up of every run, then the runs alternated over
--repeats repeats; the median of each.  The card's name and power limit are read in the same run.  One JSON line."""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from paddlerobotics_b200 import pretrain, train
from paddlerobotics_b200.agent import MujocoAgent
from train_state_cost import card

GAIT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerobotics_b200", "data", "etg_shipped_gait.npz")


def timed(main, argv):
    torch.cuda.synchronize()
    t = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        out = main(argv)
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        ckpt = os.path.join(d, "itr_1.pt")
        MujocoAgent(49, 12, seed=5).save(ckpt)
        z = np.load(GAIT)
        np.savez(os.path.join(d, "itr_1.npz"), w=z["w"], b=z["b"], param=np.zeros(12))
        runs = {}
        for n in (1, 8):
            base = ["--eval", "1", "--load", GAIT, "--eval_envs", str(n), "--task_mode", "stairstair"]
            runs["pretrain_grid_eval_envs%d" % n] = (pretrain.main, base + ["--dynamics_grid", "1"])
            runs["pretrain_plain_eval_envs%d" % n] = (pretrain.main, base)
        base = ["--eval", "1", "--load", ckpt, "--eval_envs", "8", "--task_mode", "stairstair"]
        runs["train_grid_eval_envs8"] = (train.main, base + ["--dynamics_grid", "1"])
        runs["train_plain_eval_envs8"] = (train.main, base)
        times, out = {k: [] for k in runs}, {}
        for k, (m, argv) in runs.items():
            timed(m, argv)
        for _ in range(a.repeats):
            for k, (m, argv) in runs.items():
                t, out[k] = timed(m, argv)
                times[k].append(t)
    rec = {"card": card(), "repeats": a.repeats, "wall_s": {k: float(np.median(v)) for k, v in times.items()}, "wall_s_repeats": times}
    for k, o in out.items():
        if "grid" in k:
            recs = o[:-1]
            rec[k] = {"envs": len(recs) * int(runs[k][1][runs[k][1].index("--eval_envs") + 1]), "max_mean_length": max(r["mean_length"] for r in recs),
                      "mean_length": float(np.mean([r["mean_length"] for r in recs])), "summary": o[-1]}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
