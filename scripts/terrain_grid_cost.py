"""What the terrain atlas costs on this GPU (DESIGN §8h):
    python scripts/terrain_grid_cost.py [--num_envs 4096] [--steps 200] [--eval_envs 1]
1. The float32 control step at --num_envs envs on train's eval configuration: a plain stairstair height-field handle against atlas handles
   of the stairstair grid (88 tiles) and the stairslope grid (968 tiles), env i on tile i mod T.  CUDA events around --steps steps after a
   warm-up, the three handles alternated over three repeats; the median per-step time of each.
2. The wall time of a whole pretrain --eval 1 --terrain_grid 1 of the shipped gait (the zero residual, which walks) on the stairstair and
   the stairslope grid, --eval_envs envs per geometry: set-up (tiles, create, settle), the episode of at most 601 steps and the records,
   host clock, one run each.
The card's name and power limit are read in the same run.  One JSON line."""
import argparse
import contextlib
import io
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from paddlerobotics_b200 import pretrain, train
from paddlerobotics_b200.env import VecQuadrupedalEnv
from paddlerobotics_b200.terrain import make_terrain, make_terrain_tiles, terrain_grid
from train_state_cost import card


def step_ms(env, steps, act):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        env.step(act)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--eval_envs", type=int, default=1)
    a = ap.parse_args()
    args = train.parser().parse_args([])
    cfg = train.train_env_config(args)
    cfg.pop("heightfield")
    n = a.num_envs
    _, w, b, _ = train.etg_prior()
    envs = {"plain_stairstair": VecQuadrupedalEnv(n, auto_reset=True, max_episode_steps=400, heightfield=make_terrain("stairstair"), **cfg)}
    for task, key in (("stairstair", "atlas_88"), ("stairslope", "atlas_968")):
        tiles, x0, y0, cell = make_terrain_tiles(task, terrain_grid(task))
        e = VecQuadrupedalEnv(n, auto_reset=True, max_episode_steps=400, heightfield=(tiles[0], x0, y0, cell), **cfg)
        e.set_terrain_tiles(tiles, np.arange(n, dtype=np.int32) % tiles.shape[0])
        envs[key] = e
    act = torch.zeros(n, 12, device="cuda")
    times = {k: [] for k in envs}
    for e in envs.values():
        e.reset(w, b)
        step_ms(e, 20, act)
    for _ in range(3):
        for k, e in envs.items():
            times[k].append(step_ms(e, a.steps, act))
    rec = {"card": card(), "num_envs": n, "steps": a.steps, "step_ms": {k: float(np.median(v)) for k, v in times.items()},
           "step_ms_repeats": times}
    for e in envs.values():
        e.close()
    # whole grid evaluations through the command
    gait = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerobotics_b200", "data", "etg_shipped_gait.npz")
    rec["grid_eval"] = {}
    for task in ("stairstair", "stairslope"):
        torch.cuda.synchronize()
        t = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            recs = pretrain.main(["--eval", "1", "--terrain_grid", "1", "--load", gait, "--eval_envs", str(a.eval_envs), "--task_mode", task])
        torch.cuda.synchronize()
        rec["grid_eval"][task] = {"geometries": recs[-1]["geometries"], "envs": recs[-1]["geometries"] * a.eval_envs,
                                  "wall_s": time.perf_counter() - t,
                                  "mean_length": float(np.mean([r["mean_length"] for r in recs[:-1]])),
                                  "max_mean_length": max(r["mean_length"] for r in recs[:-1]), "summary": recs[-1]}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
