"""What train and the ES phase cost across GPUs under torchrun over NCCL (DESIGN §8, multi-GPU training):
    python scripts/train_multi_cost.py [--worlds 1,2,4,8]
For each world size W that the visible GPUs allow (one rank per GPU), and for weak scaling (4096 envs per rank, a population of 64 per rank)
and strong scaling (4096 envs, a population of 64, in all):
1. the captured training iteration (--graph_iter 1, --ES 0, stairstair, batch = envs): train.main for 400 iterations, the median over
   runs of each run's median interval between log records after iteration 100, per control step, 3 runs after one warm-up run;
2. one ES generation (PopulationEvaluator, 4 rollouts per individual, 400 steps, zero residual; fitness all-gathered): 5 generations
   timed with a device synchronise after one warm-up generation, median and range.
Rank 0 prints one JSON line per (W, scaling); the card, its power limit and SM clock are read in the same run.  World sizes with fewer
GPUs than ranks are reported as not measured."""
import argparse
import json
import os
import signal
import socket
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ENVS, POP, ROLLOUTS = 4096, 64, 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()
    except Exception as e:            # the numbers stand without it, but say so
        return "unknown (%s)" % e


def iteration_us(n, iters=400):
    from paddlerobotics_b200 import train
    log = train.main(["--num_envs", str(n), "--batch", str(n), "--warmup_steps", str(4 * n), "--log_every", "50", "--ES", "0",
                      "--max_steps", str(iters * n), "--task_mode", "stairstair", "--graph_iter", "1"])
    return [n / r["interval_env_steps_per_s"] * 1e6 for r in log if r["iters"] > 100]


def es_generation_ms(pop, rank, world, dev, gens=5):
    import numpy as np
    import torch
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.es import PopulationEvaluator, SimpleGA, solutions_to_etg_device
    args = train.parser().parse_args([])
    _, w0, b0, prior = train.etg_prior()
    np.random.seed(0)
    solver = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=pop, param=np.zeros(12))
    ev = PopulationEvaluator(pop, ROLLOUTS, max_steps=400, rank=rank, world=world, device=dev, **train.env_config(args))
    out = []
    for g in range(gens + 1):
        ws, bs = solutions_to_etg_device(solver.ask(), prior, w0, b0, device=dev)
        ws, bs = ws.cpu().numpy(), bs.cpu().numpy()
        torch.cuda.synchronize(); t0 = time.perf_counter()
        fit, _ = ev.evaluate(ws, bs)
        fit = fit.double().cpu().numpy()
        dt = (time.perf_counter() - t0) * 1e3
        solver.tell(np.where(np.isfinite(fit), fit, -1e9))
        if g:
            out.append(dt)
    ev.env.close()
    return out


def worker():
    import numpy as np
    from paddlerobotics_b200 import dist_run
    rank, world, local = dist_run.ranks()
    with dist_run.process_group(world, local, "nccl") as dev:
        for scaling in ("weak", "strong"):
            n = ENVS * world if scaling == "weak" else ENVS
            pop = POP * world if scaling == "weak" else POP
            iteration_us(n)                                  # warm-up run
            runs = [float(np.median(iteration_us(n))) for _ in range(3)]
            gen = es_generation_ms(pop, rank, world, dev)
            if rank == 0:
                print("RESULT " + json.dumps({"world": world, "scaling": scaling, "envs": n, "popsize": pop, "rollouts": ROLLOUTS,
                                              "iteration_us": {"median": float(np.median(runs)), "runs": runs},
                                              "es_generation_ms": {"median": float(np.median(gen)), "min": min(gen), "max": max(gen)}}), flush=True)


def main():
    import torch
    p = argparse.ArgumentParser()
    p.add_argument("--worlds", type=str, default="1,2,4,8")
    a = p.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for world in (int(x) for x in a.worlds.split(",")):
        if world > torch.cuda.device_count():
            print(json.dumps({"world": world, "result": "not measured: %d GPUs visible" % torch.cuda.device_count()}), flush=True)
            continue
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        # the launcher in a session of its own, so that a timeout kills its ranks too, not the launcher alone
        proc = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % world, "--master-addr",
                                 "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__)], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                text=True, start_new_session=True)
        try:
            stdout, stderr = proc.communicate(timeout=3600)
        finally:
            try:
                os.killpg(proc.pid, signal.SIGKILL)
            except ProcessLookupError:
                pass
            proc.wait()
        for line in stdout.splitlines():
            if line.startswith("RESULT "):
                print(line[7:], flush=True)
        if proc.returncode != 0:
            print(json.dumps({"world": world, "error": stderr[-2000:]}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    worker() if "RANK" in os.environ else main()
