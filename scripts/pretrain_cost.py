"""Cost of an ETG-pretraining generation (paddlerobotics_b200.pretrain) at the reference's population (40) and at 4096, on stairstair, and the
control-step time of train.py --eval with the fused episode-statistics kernel against the 1 + 6 launch loop it replaced.  Prints one JSON line
per population with the card's name and power limit read in the same run; every time is the median of --gens generations (after one warm-up):

  * ask_s / tell_s: host clock around SimpleGA.ask / tell;
  * fit_gpu_s: CUDA events around solutions_to_etg_device (b2q_etg_fit, one thread per individual, float64);
  * evaluate_gpu_s: CUDA events around PopulationEvaluator.evaluate(terms=EVAL_TERMS) (reset, up to 401 control steps, the per-step fused
    accumulator, the end-of-generation reductions); evaluate_plain_gpu_s the same call without terms (b2q_es_accumulate per step);
  * generation_s: host clock around the whole generation (ask, fit, evaluate, reading the fitness back, tell);
  * eval_step_fused_ms / eval_step_old_ms: CUDA events around --steps control steps of the --eval loop (policy forward, env step, statistics)
    with b2q_es_accumulate_terms and with the old index_select + copies + 7 b2q_es_accumulate launches, alternated --reps times, per step.

    python scripts/pretrain_cost.py [--gens 5] [--popsizes 40 4096]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paddlerobotics_b200 import _lib, pretrain  # noqa: E402
from paddlerobotics_b200._config import INFO  # noqa: E402
from paddlerobotics_b200.agent import MujocoAgent  # noqa: E402
from paddlerobotics_b200.env import VecQuadrupedalEnv  # noqa: E402
from paddlerobotics_b200.es import EpisodeStats, PopulationEvaluator, SimpleGA, solutions_to_etg_device  # noqa: E402
from paddlerobotics_b200.train import EVAL_TERMS, etg_prior  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:     # the number is still reported, with the reason the card's limits are unknown
        return "nvidia-smi unavailable (%s)" % e


def generation_costs(pop, gens, cfg, prior, w0, b0):
    np.random.seed(0)
    ga = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=pop, param=np.zeros(12))
    ev = PopulationEvaluator(pop, 1, max_steps=pretrain.ES_MAX_STEP + 1, policy=None, **cfg)
    ev_ = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    rec = {k: [] for k in ("ask_s", "fit_gpu_s", "evaluate_gpu_s", "evaluate_plain_gpu_s", "tell_s", "generation_s", "mean_len")}
    for g in range(gens + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sol = ga.ask()
        t1 = time.perf_counter()
        ev_[0].record()
        ws, bs = [x.cpu().numpy() for x in solutions_to_etg_device(sol, prior, w0, b0)]
        ev_[1].record()
        fit, mlen, _, _ = ev.evaluate(ws, bs, terms=EVAL_TERMS)
        ev_[2].record()
        f = fit.double().cpu().numpy()
        t2 = time.perf_counter()
        ga.tell(np.where(np.isfinite(f), f, -1e9))
        t3 = time.perf_counter()
        ev_[3].record()
        ev.evaluate(ws, bs)                                     # the same generation without the term statistics, for comparison
        ev_[4].record()
        torch.cuda.synchronize()
        if g == 0:
            continue
        rec["ask_s"].append(t1 - t0); rec["tell_s"].append(t3 - t2); rec["generation_s"].append(t3 - t0)
        rec["fit_gpu_s"].append(ev_[0].elapsed_time(ev_[1]) * 1e-3); rec["evaluate_gpu_s"].append(ev_[1].elapsed_time(ev_[2]) * 1e-3)
        rec["evaluate_plain_gpu_s"].append(ev_[3].elapsed_time(ev_[4]) * 1e-3); rec["mean_len"].append(float(mlen.double().mean()))
    ev.env.close()
    return {k: float(np.median(v)) for k, v in rec.items()}


def eval_step_costs(n, steps, reps, cfg, w, b):
    """ms per control step of the --eval loop, fused statistics against the old per-term loop, alternated."""
    lib = _lib.load()
    agent = MujocoAgent(49, 12, seed=0)
    env = VecQuadrupedalEnv(n, auto_reset=False, **cfg)
    dev, es, stream = env.device, env.obs.element_size(), env._stream()
    nt = len(EVAL_TERMS)
    stats = EpisodeStats(lib, n, env.dtype, dev, EVAL_TERMS)
    cols = torch.tensor([INFO[k] for k in EVAL_TERMS], device=dev)
    alive = torch.ones(n, dtype=torch.uint8, device=dev)
    ret, length = torch.zeros(n, dtype=env.dtype, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    t_alive, t_sum, t_len = torch.empty(nt, n, dtype=torch.uint8, device=dev), torch.zeros(nt, n, dtype=env.dtype, device=dev), torch.zeros(nt, n, dtype=torch.int32, device=dev)
    t_val = torch.empty(nt, n, dtype=env.dtype, device=dev)

    def fused(info, rew, done):
        stats.step(rew, done, info, stream)

    def old(info, rew, done):
        t_val.copy_(info.index_select(1, cols).T)
        t_alive.copy_(alive.expand(nt, n))
        for j in range(nt):
            assert lib.b2q_es_accumulate(t_val[j].data_ptr(), done.data_ptr(), t_alive[j].data_ptr(), t_sum[j].data_ptr(), t_len[j].data_ptr(), n, es, stream) == 0
        assert lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), alive.data_ptr(), ret.data_ptr(), length.data_ptr(), n, es, stream) == 0

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {"fused": [], "old": []}
    for rep in range(reps + 1):
        for name, acc in (("fused", fused), ("old", old)):
            obs = env.reset(w, b)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                obs, rew, done, info = env.step(agent.predict_batch(obs) * 0.3, donef=False)
                acc(info, rew, done)
            e1.record()
            torch.cuda.synchronize()
            if rep:
                out[name].append(e0.elapsed_time(e1) / steps)
    env.close()
    return {"eval_step_fused_ms": float(np.median(out["fused"])), "eval_step_old_ms": float(np.median(out["old"])),
            "eval_step_fused_ms_spread": [min(out["fused"]), max(out["fused"])], "eval_step_old_ms_spread": [min(out["old"]), max(out["old"])]}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--gens", type=int, default=5, help="timed generations per population (after one warm-up)")
    p.add_argument("--popsizes", type=int, nargs="+", default=[40, 4096])
    p.add_argument("--steps", type=int, default=200, help="control steps per timed --eval window")
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--task_mode", type=str, default="stairstair")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pretrain_cost.py measures on the GPU: no CUDA device")
    cfg = pretrain.env_config(pretrain.parser().parse_args(["--task_mode", args.task_mode]))
    _, w0, b0, prior = etg_prior()
    info, name = gpu_info(), torch.cuda.get_device_name(0)
    for pop in args.popsizes:
        out = {"popsize": pop, "task_mode": args.task_mode, "gens": args.gens}
        out.update(generation_costs(pop, args.gens, cfg, prior, w0, b0))
        out["eval_envs"] = pop
        out.update(eval_step_costs(pop, args.steps, args.reps, cfg, w0, b0))
        out["device"], out["nvidia_smi"] = name, info
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
