"""Cost of one camera-image call (VecQuadrupedalEnv.get_camera_image, the b2q_render kernel plus the state read and the follow-camera
matrices) at V = 1, 16 and 64 views of 640 x 480 on `stairstair`, float32, timed with CUDA events.  The sizes are warmed up first and
then alternated inside one run, so they see the same clocks.  Prints one JSON line per size plus the card's name and power limit.

    python scripts/render_cost.py [--reps 20] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paddlerobotics_b200.env import VecQuadrupedalEnv  # noqa: E402
from paddlerobotics_b200.etg import ETG_layer, Opt_with_points  # noqa: E402
from paddlerobotics_b200.terrain import make_terrain  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:     # the number is still reported, with the reason the card's limits are unknown
        return "nvidia-smi unavailable (%s)" % e


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--width", type=int, default=640)
    p.add_argument("--height", type=int, default=480)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_cost.py measures on the GPU: no CUDA device")
    sizes = (1, 16, 64)
    env = VecQuadrupedalEnv(max(sizes), heightfield=make_terrain("stairstair"))
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    env.reset(w, b, x_offset=np.linspace(0.0, 2.0, max(sizes)))       # robots spread along the approach and the stairs
    zero = torch.zeros(max(sizes), 12, device=env.device)
    for _ in range(20):
        env.step(zero)
    ids = {V: torch.arange(V, dtype=torch.int32, device=env.device) for V in sizes}
    for V in sizes:                       # warm-up of every size (buffers, constants, module load)
        for _ in range(3):
            env.get_camera_image(args.width, args.height, env_ids=ids[V])
    torch.cuda.synchronize()
    times = {V: [] for V in sizes}
    for _ in range(args.rounds):
        for V in sizes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                env.get_camera_image(args.width, args.height, env_ids=ids[V])
            e1.record()
            torch.cuda.synchronize()
            times[V].append(e0.elapsed_time(e1) / args.reps)
    info = gpu_info()
    for V in sizes:
        ms = float(np.median(times[V]))
        rec = {"views": V, "width": args.width, "height": args.height, "terrain": "stairstair", "precision": "f32", "ms_per_call": ms,
               "ms_spread": [float(min(times[V])), float(max(times[V]))], "mpixel_per_s": V * args.width * args.height / (ms * 1e-3) / 1e6,
               "device": torch.cuda.get_device_name(env.device), "nvidia_smi": info}
        print(json.dumps(rec), flush=True)
    env.close()


if __name__ == "__main__":
    main()
