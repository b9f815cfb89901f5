"""Generates tests/golden/bezier_gait.npz: the reference's open-loop Bezier gait (deployment --gait 1) from the UNMODIFIED
deployment/utilities/Bezier.py, SpotOL.py and robots/a1.py, imported through oracle/ref_shim.py.

It drives GaitWrapper.step's exact parameter path (deployment/envs/EnvWrapper.py:155-190): BezierStepper.StateMachine(), the forced
ClearanceHeight and the six clips, the `timesteps > 5` switch to GenerateTrajectoryX(0, 0, 0, 1, ...), and the A1 IK of each foot.
Two things differ from the wrapper and are not gait arithmetic: the contacts come from the case's stream, not from `info` (which
the wrapper never updates, EnvWrapper.py:193), and T_b0 is a1.foot_positions_in_base_frame of the case's pose (GetFootPositionsInBaseFrame
of a settled robot).  NumPy 2 has no np.math, which BezierGait.Binomial calls: it is pointed at the math module here.

Run where the reference is installed:  python tests/golden/make_bezier_golden.py
"""
import copy
import math
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_shim  # noqa: E402

STEPS = 300
DT = 0.026           # test.py --dt
VELOCITY = 0.5       # GaitWrapper(velocity=0.5)
POSE = np.array([0, 0.9, -1.8] * 4)


def poses():
    """The nominal pose and two perturbed ones; the second has nearly straight knees, so some swing feet leave the leg's reach."""
    rng = np.random.default_rng(7)
    p1 = POSE + rng.uniform(-0.15, 0.15, 12)
    p2 = np.array([0.05, 0.15, -0.3, -0.05, 0.1, -0.25, 0.08, 0.2, -0.35, -0.02, 0.05, -0.2])
    return np.stack([POSE, p1, p2])


def contact_streams():
    """[cases, STEPS] bits of the reference foot: all 0, all 1, one-step touches every 14 steps at four offsets (so the touch lands
    at different phases of the 0.36 s stride), two-step touches every 9 steps, and two seeded random streams."""
    s = np.arange(STEPS)
    rows = [np.zeros(STEPS), np.ones(STEPS)]
    rows += [((s % 14) == o).astype(float) for o in (0, 3, 7, 11)]
    rows.append(((s % 9) < 2).astype(float))
    for seed in (1, 2):
        rows.append(np.random.default_rng(seed).integers(0, 2, STEPS).astype(float))
    return np.stack(rows).astype(np.uint8)


def run_case(Bezier, SpotOL, a1, q, contacts):
    """GaitWrapper.reset + STEPS x GaitWrapper.step's gait arithmetic (EnvWrapper.py:140-190)."""
    bz_step = SpotOL.BezierStepper(dt=DT, StepVelocity=VELOCITY)
    bzg = Bezier.BezierGait(dt=DT)
    T_b0_ = copy.copy(a1.foot_positions_in_base_frame(q))
    T_b0 = {"FL": T_b0_[0, :], "FR": T_b0_[1, :], "BL": T_b0_[2, :], "BR": T_b0_[3, :]}
    feet, ang, flags = np.zeros((STEPS, 4, 3)), np.zeros((STEPS, 12)), np.zeros((STEPS, 3))
    timesteps = 0
    for i in range(STEPS):
        timesteps += 1
        pos, orn, StepLength, LateralFraction, YawRate, StepVelocity, ClearanceHeight, PenetrationDepth = bz_step.StateMachine()
        ClearanceHeight = 0.05
        StepLength = np.clip(StepLength, bz_step.StepLength_LIMITS[0], bz_step.StepLength_LIMITS[1])
        StepVelocity = np.clip(StepVelocity, bz_step.StepVelocity_LIMITS[0], bz_step.StepVelocity_LIMITS[1])
        LateralFraction = np.clip(LateralFraction, bz_step.LateralFraction_LIMITS[0], bz_step.LateralFraction_LIMITS[1])
        YawRate = np.clip(YawRate, bz_step.YawRate_LIMITS[0], bz_step.YawRate_LIMITS[1])
        ClearanceHeight = np.clip(ClearanceHeight, bz_step.ClearanceHeight_LIMITS[0], bz_step.ClearanceHeight_LIMITS[1])
        PenetrationDepth = np.clip(PenetrationDepth, bz_step.PenetrationDepth_LIMITS[0], bz_step.PenetrationDepth_LIMITS[1])
        c = [int(contacts[i]), 0, 0, 0]
        if timesteps > 5:
            T_bf = bzg.GenerateTrajectoryX(StepLength, LateralFraction, YawRate, StepVelocity, T_b0, ClearanceHeight, PenetrationDepth, c)
        else:
            T_bf = bzg.GenerateTrajectoryX(0.0, 0.0, 0.0, 1, T_b0, ClearanceHeight, PenetrationDepth, c)
        for leg, key in enumerate(T_bf):
            feet[i, leg] = T_bf[key]
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")      # arccos of an unreachable foot: NaN, as the reference gives
                ang[i, 3 * leg:3 * leg + 3] = a1.foot_position_in_hip_frame_to_joint_angle(T_bf[key] - a1.HIP_OFFSETS[leg], (-1) ** (leg + 1))
        flags[i] = (float(bzg.TD), float(bzg.SwRef), float(bzg.StanceSwing))
    return T_b0_, feet, ang, flags


def main():
    ns = ref_shim.load()
    np.math = math                                   # NumPy 2 shim for BezierGait.Binomial (Bezier.py:206-208)
    from utilities import Bezier, SpotOL
    q, c = poses(), contact_streams()
    qs, cs, tb0, feet, ang, flags = [], [], [], [], [], []
    for qi in q:
        for ci in c:
            t, f, a, fl = run_case(Bezier, SpotOL, ns.a1, qi, ci)
            qs.append(qi); cs.append(ci); tb0.append(t); feet.append(f); ang.append(a); flags.append(fl)
    out = {"q": np.stack(qs), "contact": np.stack(cs), "tb0": np.stack(tb0), "feet": np.stack(feet), "ang": np.stack(ang),
           "td": np.stack(flags)[..., 0], "swref": np.stack(flags)[..., 1], "swing": np.stack(flags)[..., 2]}
    path = os.path.join(HERE, "bezier_gait.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d cases x %d steps, %d NaN joint angles" % (path, out["q"].shape[0], STEPS, int(np.isnan(out["ang"]).sum())))


if __name__ == "__main__":
    main()
