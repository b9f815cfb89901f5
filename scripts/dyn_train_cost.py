"""Cost of a dynamics-identification epoch (paddlerobotics_b200.dynamic_train): ask, evaluate, tell and save, at the reference's population
(K 20 x thread 2 = 40) and at 4096, on synthetic data (the shipped CPG table as the gait tables, random statistics).  Prints one JSON line
per population with the card's name and power limit read in the same run:

  * epoch_s: host clock around the whole epoch (ask, evaluate, reading the rewards back, tell, np.save);
  * evaluate_gpu_s: CUDA events around DynamicsEvaluator.evaluate (the settle under new dynamics, 100 steps of the step kernel and the
    loss kernels, and any gap in between);
  * evaluate_enqueue_s: host clock from the call to its return, before the rewards are read back.  When it approaches evaluate_gpu_s
    the host, not the GPU, sets the pace;
  * map_s: of that, the host's mapping of the population to dynamics rows (etg.param2dynamic_rows), and map_per_row_s the per-individual
    param2dynamic_dict -> dynamic_dict_to_row it replaces (same rows, bit for bit);
  * settle_gpu_s: CUDA events around the set_dynamics (which settles every env under its new dynamics) and reset of one evaluation.

    python scripts/dyn_train_cost.py [--epochs 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paddlerobotics_b200.dynamic_train import STEPS, evaluator_config, make_solver  # noqa: E402
from paddlerobotics_b200.es import DynamicsEvaluator  # noqa: E402
from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict, param2dynamic_rows  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:     # the number is still reported, with the reason the card's limits are unknown
        return "nvidia-smi unavailable (%s)" % e


def synthetic_data():
    pose = np.array([0, 0.9, -1.8] * 4)
    tab = np.load(os.path.join(ROOT, "tests", "golden", "gait_action_list_CPG_stairstair7_12_3.npy")) + pose
    rng = np.random.default_rng(0)
    gait, md = {"exp": tab[:STEPS], "ori": tab[STEPS:2 * STEPS]}, {}
    for k in gait:
        md[k + "_motor_mean"], md[k + "_motor_std"] = gait[k] + rng.normal(0, 0.02, (STEPS, 12)), rng.uniform(0.05, 0.1, (STEPS, 12))
        md[k + "_drpy_mean"], md[k + "_drpy_std"] = rng.normal(0, 0.2, (STEPS, 3)), rng.uniform(0.3, 0.6, (STEPS, 3))
    return gait, md


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=5, help="timed epochs per population (after one warm-up epoch)")
    p.add_argument("--popsizes", type=int, nargs="+", default=[40, 4096])
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dyn_train_cost.py measures on the GPU: no CUDA device")
    gait, md = synthetic_data()
    info, name = gpu_info(), torch.cuda.get_device_name(0)
    with tempfile.TemporaryDirectory() as outdir:
        for pop in args.popsizes:
            np.random.seed(0)
            solver = make_solver("ga", pop, 0.1)
            ev = DynamicsEvaluator(pop, gait, md, keys=("exp", "ori"), steps=STEPS, **evaluator_config())
            rec = {k: [] for k in ("epoch_s", "ask_s", "evaluate_enqueue_s", "evaluate_gpu_s", "tell_s", "save_s", "map_s", "map_per_row_s", "settle_gpu_s")}
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for epoch in range(args.epochs + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                sol = solver.ask()
                t1 = time.perf_counter()
                e0.record()
                r = ev.evaluate(sol)
                e1.record()
                t2 = time.perf_counter()
                rewards = r.double().cpu().numpy()
                t3 = time.perf_counter()
                solver.tell(rewards)
                t4 = time.perf_counter()
                np.save(os.path.join(outdir, "dynamic_param%d.npy" % epoch), solver.result()[0])
                t5 = time.perf_counter()
                if epoch == 0:
                    continue                                  # warm-up: module load, first allocations
                rec["epoch_s"].append(t5 - t0); rec["ask_s"].append(t1 - t0); rec["evaluate_enqueue_s"].append(t2 - t1)
                rec["evaluate_gpu_s"].append(e0.elapsed_time(e1) * 1e-3); rec["tell_s"].append(t4 - t3); rec["save_s"].append(t5 - t4)
                tm = time.perf_counter()
                rows = param2dynamic_rows(sol)
                rec["map_s"].append(time.perf_counter() - tm)
                tm = time.perf_counter()
                np.array([dynamic_dict_to_row(param2dynamic_dict(s)) for s in sol])
                rec["map_per_row_s"].append(time.perf_counter() - tm)
                torch.cuda.synchronize()
                e0.record()
                ev.env.set_dynamics(np.tile(rows, (2, 1)))
                ev.env.reset()
                e1.record()
                torch.cuda.synchronize()
                rec["settle_gpu_s"].append(e0.elapsed_time(e1) * 1e-3)
            ev.env.close()
            out = {"popsize": pop, "envs": 2 * pop, "control_steps": STEPS, "epochs": args.epochs}
            out.update({k: float(np.median(v)) for k, v in rec.items()})
            out["epoch_s_spread"] = [min(rec["epoch_s"]), max(rec["epoch_s"])]
            out["device"], out["nvidia_smi"] = name, info
            print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
