"""Deployment rehearsal with the reference's open-loop Bezier gait — deployment/test.py run with `--gait 1` (GaitWrapper,
deployment/envs/EnvWrapper.py:123-193), on the GPU.

Same flags, defaults, batch layout, outputs and refusals as deploy_test (test.py's flags, :108-126), with the Bezier trot added: its IK
joint angles replace the base pose, so step i applies IK(feet_i) + 0.3 * student(obs) + table[i], with the touchdown of the gait's
reference foot read from the observation's FootContactSensor block (deploy.py, DESIGN §8f).  data/{suffix}_rpm.npz keeps test.py's
action_list meaning (student + table, without the gait), and each JSON line carries "gait": 1.  Any non-zero --gait (default 1) runs
the gait, as test.py's `if gait:`; --gait 0 is deploy_test itself.

Refused before any device work, besides deploy_test's refusals: the gait with --sensor_contact 0 (the reference raises KeyError on
info["FootContactSensor"]) and with --enable_action_filter 1 (the reference filters the action before the gait's angles are added, the
engine's filter acts on the whole joint target).

    python -m paddlerobotics_b200.deploy_bezier --load student.pt --ETG_path gait.npy --max_time 5 --x_starts 8
"""
import argparse
import json
import os

import numpy as np

from . import deploy_test
from .deploy import deploy_config, rehearse
from .env import VecQuadrupedalEnv


def parser():
    p = deploy_test.parser()
    p.description = __doc__.split("\n")[0]
    p.set_defaults(gait=1)
    return p


def check_args(args):
    """Everything the gait rehearsal refuses, before any device work.  Returns (table, student state dict)."""
    if not args.sensor_contact:
        raise ValueError("--gait %d with --sensor_contact 0: the Bezier gait reads the foot contacts (the reference raises KeyError on "
                         "info['FootContactSensor'])" % args.gait)
    if args.enable_action_filter:
        raise NotImplementedError("--gait %d with --enable_action_filter 1: the reference filters the action before the Bezier gait adds its "
                                  "angles, the engine's filter acts on the whole joint target" % args.gait)
    rest = argparse.Namespace(**vars(args))
    rest.gait = 0                                   # the remaining checks are deploy_test's
    return deploy_test.check_args(rest)


def main(argv=None):
    from .agent import MujocoAgent
    args = parser().parse_args(argv)
    if not args.gait:                               # only an explicit --gait 0 gets here: the same arguments mean the same to deploy_test
        return deploy_test.main(argv)
    table, sd = check_args(args)
    steps = deploy_test.steps_of(args)
    dyn, labels = deploy_test.group_rows(args.dynamic_param)
    group, xoff = deploy_test.batch_layout(len(labels), args.x_starts)
    env = VecQuadrupedalEnv(len(group), auto_reset=False, **deploy_config(args))
    if args.dynamic_param:
        env.set_dynamics(dyn[group])
    student = MujocoAgent(int(sd["actor_model.l1.weight"].shape[1]), 12)
    student.load_state_dict(sd)
    res = rehearse(env, student, table, steps, act_bound=deploy_test.ACT_BOUND, x_offset=xoff, gait=True)
    env.close()
    os.makedirs("data", exist_ok=True)
    np.savez(os.path.join("data", args.suffix + "_rpm.npz"), action=res["action"], obs=res["obs"])      # test.py:105
    recs = deploy_test.summarise(res, group, labels)
    for r in recs:
        r["gait"] = 1
        print(json.dumps(r), flush=True)
    return recs, res


if __name__ == "__main__":
    main()
