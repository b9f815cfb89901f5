"""The gait-table export of ETGRL/env_test.py: 600 zero-residual control steps of make_env(..., ETG_path=load) and, with --save 1, the table of
info["ETG_act"] in gait_action_list_ETG_{suffix}.npy in the current directory: the `.npy` gait that deployment reads (README §3).

    python -m paddlerobotics_b200.env_test --load pretrain_log/exp0/itr_160400.npz --save 1 --suffix stair

Deviations: the reference reads its dynamics from a fixed data file; here --dynamic_param PATH.npy sets them and the default is nominal.
The reference opens a GUI window (render=True); here nothing is drawn and --video is accepted and ignored, as it is in the reference.
"""
import argparse
import os

import numpy as np

STEPS = 600                 # env_test.py:51


def parser():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    # ---- env_test.py:31-38
    p.add_argument("--load", type=str, default="data/origin_ETG/ESStair_origin.npz", help="the gait (.npz with w, b)")
    p.add_argument("--video", type=int, default=0, help="accepted and ignored, as in the reference")
    p.add_argument("--task", type=str, default="stairstair")
    p.add_argument("--suffix", type=str, default="exp")
    p.add_argument("--save", type=int, default=0, help="1: write gait_action_list_ETG_{suffix}.npy")
    p.add_argument("--step_y", type=float, default=0.05)
    # ---- the data file of env_test.py:40-41
    p.add_argument("--dynamic_param", type=str, default="", help="PATH.npy: a 48-vector in [-1, 1] -> param2dynamic_dict; empty = nominal dynamics")
    return p


def main(argv=None):
    """Returns the [600, 12] table (and writes it with --save 1)."""
    p = parser()
    args = p.parse_args(argv)
    if not (args.load.endswith(".npz") and os.path.isfile(args.load)):
        p.error("--load %s: the gait must be an existing .npz with w and b" % args.load)
    from .env import make_env
    from .etg import param2dynamic_dict
    dyn = param2dynamic_dict(np.load(args.dynamic_param).reshape(-1)) if args.dynamic_param else None
    # reward_param: the reference passes MonitorEnv's default dict; the ETG_act table does not depend on reward weights, so the engine's are kept
    # float64, as the reference computes: over 600 steps a float32 ETG clock drifts by ~1e-5 rad in the table
    env = make_env("Quadrupedal", task=args.task, dynamic_param=dyn, normal=1, ETG=1, ETG_path=args.load, step_y=args.step_y, precision="f64")
    env.reset()
    table = []
    for _ in range(STEPS):
        _, _, _, info = env.step(np.zeros(12), donef=False)
        table.append(info["ETG_act"])
    env.close()
    table = np.array(table)
    if args.save:
        np.save("gait_action_list_ETG_{}.npy".format(args.suffix), table)
    return table


if __name__ == "__main__":
    main()
