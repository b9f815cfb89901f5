"""What storing the ES rollouts in the replay memory (train.py --es_rpm 1) costs: one ES generation at the bench's ES workload
(256 individuals x 16 rollouts x 400 control steps, zero residual action as in bench.py) timed with and without
`PopulationEvaluator.evaluate(..., replay=)`, alternating the two in one run.  Prints the card's name and power limit with the numbers.

    python scripts/es_rpm_cost.py [--gens 5] [--out /tmp/es_rpm_cost.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from paddlerobotics_b200.es import PopulationEvaluator, SimpleGA, solutions_to_etg_device
from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
from paddlerobotics_b200.replay import ReplayMemory


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--gens", type=int, default=5, help="timed generations per arm")
    p.add_argument("--out", type=str, default="")
    args = p.parse_args()
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    pop, roll, T = 256, 16, 400
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w0, b0, pts = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    np.random.seed(0)
    ga = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=pop, param=np.zeros(12))
    ev = PopulationEvaluator(pop, roll, max_steps=T)
    rpm = ReplayMemory(1000000, 49, 12, device_cursor=True)          # the training loop's default memory and cursor mode
    times = {"without": [], "with": []}
    rows = []
    for gi in range(2 * args.gens + 2):                                # the first pair warms both arms up
        arm = "with" if gi % 2 else "without"
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sol = ga.ask()
        wsd, bsd = solutions_to_etg_device(sol, pts, w0, b0)
        fit, mlen = ev.evaluate(wsd.cpu().numpy(), bsd.cpu().numpy(), replay=rpm if arm == "with" else None)
        ga.tell(fit.double().cpu().numpy())
        if arm == "with":
            rpm.sync_host()                                            # what train.py does after the phase
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if gi >= 2:
            times[arm].append(dt)
            if arm == "with":
                rows.append(int(ev.rows))
    res = {"card": card, "popsize": pop, "rollouts": roll, "steps": T, "generations_per_arm": args.gens,
           "s_per_generation_without_replay": float(np.median(times["without"])), "s_per_generation_with_replay": float(np.median(times["with"])),
           "all_s_without": times["without"], "all_s_with": times["with"], "rows_appended_per_generation": rows}
    res["overhead_frac"] = res["s_per_generation_with_replay"] / res["s_per_generation_without_replay"] - 1.0
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
