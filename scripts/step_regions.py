"""Where do the step kernel's cycles go?  Region clocks of b2q_step_kernel<float, 0> on the bench workload.

Builds the library with -DB2Q_REGION_CLOCKS into its own path (never csrc/libb2q.so, whose step kernel has no clock reads), runs
bench.py's flagship workload through it (4096 envs, flat terrain, the Opt_with_points(0.1, 0.05) ETG, uniform +-0.3 residuals,
auto-reset, L2 flushed between steps) and reads back one row per warp: the cycles lane 0 spent in each region, summed over the timed
steps.  Regions (b2q_sim.cuh, RC_*): prologue (model staging, state and parameter loads); per substep, before the PGS sweep, PD and
kinematics, bias forces and composite inertias, Schur reduction and Cholesky, contact rows and the Delassus exchange (reported together
as pre_sweep too); the sweep, the impulse application and integration after it, the loop between substeps (observation-ring writes),
and the epilogue (ETG, observation, reward, auto-reset, stores).

These are INSTRUMENTED numbers: the clock reads cost a few cycles each and constrain the scheduling around them.  The step time users
get is the one bench.py reports from the product library.

  python scripts/step_regions.py [--lib PATH] [--src DIR] [--steps 400] [--warmup 40] [--json PATH]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

REGIONS = ["prologue", "pd_kinematics", "bias_inertia", "schur_cholesky", "contact_rows", "delassus_exchange",
           "sweep", "post_sweep", "between_substeps", "epilogue"]                              # RC_* order of b2q_sim.cuh
PRE_SWEEP = REGIONS[1:6]                                                                     # the substep's part before the sweep
COLS = len(REGIONS) + 2                                                                       # + entry-to-exit cycles, launches


def build_instrumented(lib, src):
    from paddlerobotics_b200 import build as b
    srcs = [os.path.join(src, s) for s in b.SOURCES]
    deps = srcs + [os.path.join(src, h) for h in b.HEADERS]
    if os.path.exists(lib) and all(os.path.getmtime(p) <= os.path.getmtime(lib) for p in deps if os.path.exists(p)):
        return lib
    os.makedirs(os.path.dirname(os.path.abspath(lib)), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + b.NVCC_FLAGS + ["-DB2Q_REGION_CLOCKS", "-o", lib] + srcs)
    return lib


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout
        name, pl, mx = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit": pl, "sm_max_clock": mx}
    except Exception as ex:
        return {"error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "build", "region_clocks", "libb2q.so"), help="instrumented library (built here if missing or stale)")
    ap.add_argument("--src", default=os.path.join(ROOT, "paddlerobotics_b200", "csrc"), help="CUDA sources to build it from")
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()

    lib_path = build_instrumented(os.path.abspath(args.lib), args.src)
    import torch
    from paddlerobotics_b200 import _lib
    _lib._LIB_PATH, _lib._lib = lib_path, None          # the env below binds the instrumented library
    lib = _lib.load()
    rc_fn = lib.b2q_region_clocks                         # AttributeError: not a region-clock build
    rc_fn.restype, rc_fn.argtypes = C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int]
    from bench import ClockSampler, ENVS_PER_GPU, etg_weights
    from paddlerobotics_b200.env import VecQuadrupedalEnv

    n, K, W = ENVS_PER_GPU, args.steps, args.warmup
    w, b = etg_weights()
    env = VecQuadrupedalEnv(n, device=0, auto_reset=True)
    env.reset(w, b)
    dev = env.device
    g = torch.Generator(device=dev); g.manual_seed(1234)
    pool = torch.rand(64, n, 12, device=dev, generator=g) * 0.6 - 0.3
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev, dtype=torch.float32)
    for k in range(W):
        env.step(pool[k % 64])
    assert rc_fn(0, None, 0, 1) == 0
    sampler = ClockSampler(0); sampler.start()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    for k in range(K):
        flush.zero_()
        ev[k][0].record(); env.step(pool[(W + k) % 64]); ev[k][1].record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    us = 1e3 * sum(a.elapsed_time(c) for a, c in ev) / K
    warps = (n * 4 + 31) // 32
    rows = np.zeros((warps, COLS), dtype=np.uint64)
    assert rc_fn(0, rows.ctypes.data, warps, 0) == 0
    R, iters = int(env.cfg.action_repeat), int(env.cfg.solver_iters)
    env.close()

    assert (rows[:, -1] == K).all(), "every warp must have run every timed step"
    per_step = rows[:, :-1].astype(np.float64) / K                 # [warps][regions + total] cycles per control step
    total = per_step[:, -1]
    res = {"instrumented": True, "kernel": "b2q_step_kernel<float, 0>", "envs": n, "warps": warps, "steps": K, "warmup": W,
           "substeps": R, "sweeps_per_substep": iters, "rows_per_sweep": 12, "lib": lib_path,
           "card": card(), "clocks_during_timed_steps": clocks, "us_per_step_instrumented": us, "regions": {}}
    cols = {name: per_step[:, i] for i, name in enumerate(REGIONS)}
    cols["pre_sweep"] = sum(cols[name] for name in PRE_SWEEP)
    cols["total"] = total
    for name, c in cols.items():
        res["regions"][name] = {"median": float(np.median(c)), "max": float(c.max()), "share": float(c.sum() / total.sum())}
    sw = per_step[:, REGIONS.index("sweep")]
    res["sweep_cycles_per_sweep"] = {"median": float(np.median(sw)) / (R * iters), "max": float(sw.max()) / (R * iters)}
    res["sweep_cycles_per_row"] = {"median": float(np.median(sw)) / (R * iters * 12), "max": float(sw.max()) / (R * iters * 12)}

    print("INSTRUMENTED region clocks (clock64 reads in the kernel; bench.py's product library has none and is the headline timing)")
    print("card: %s | SM clock during the timed steps: median %s MHz (max %s), throttle reasons %s" %
          (res["card"], clocks.get("sm_mhz"), clocks.get("sm_max_mhz"), clocks.get("reasons")))
    print("%d envs = %d warps, %d timed steps after %d warm-up; %.1f us per step with the clock reads" % (n, warps, K, W, us))
    print("%-18s %14s %14s %8s" % ("region", "median cyc", "max cyc", "share"))
    for name, v in res["regions"].items():
        print("%-18s %14.0f %14.0f %7.1f%%" % (name, v["median"], v["max"], 100 * v["share"]))
    print("sweep: %.1f cycles per nominal sweep, %.2f per row (median warp; over %d substeps x %d sweeps x 12 rows per step, although the exact early exit runs fewer)" %
          (res["sweep_cycles_per_sweep"]["median"], res["sweep_cycles_per_row"]["median"], R, iters))
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
