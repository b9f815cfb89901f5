import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    return np.load(os.path.join(GOLDEN, "reference_vectors.npz"))


@pytest.fixture(scope="session")
def etg_default(golden):
    """W,b of Opt_with_points(Footheight=0.1, Steplength=0.05) as produced by the reference's own train.py code."""
    return golden["opt_w0"], golden["opt_b0"]


@pytest.fixture(scope="session")
def etg_stable():
    """A gentler gait (Footheight 0.03, Steplength 0.02) that walks >1000 steps open-loop: long-horizon drift tests."""
    from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.03, Steplength=0.02)
    return w, b


def fit_etg_from_table(table, t0):
    """W,b of the ETG whose info['ETG_act'] table this is (least squares through the pinned FK; sample k is t0 + 0.026 k)."""
    from oracle import oracle as O
    from paddlerobotics_b200 import etg as E
    cfg = O.default_config()
    ts = t0 + 0.026 * np.arange(table.shape[0])
    pose = np.array([0, .9, -1.8] * 4)
    A, Y = [], []
    for k in range(table.shape[0]):
        q = table[k] + pose
        for leg in (0, 1):
            foot = O.fk_leg(q[3 * leg:3 * leg + 3], (-1) ** (leg + 1)) + E.HIP_OFFSETS[leg]
            A.append(np.concatenate([O.etg_features(cfg, ts[k] if leg == 0 else ts[k] + 0.25), [1.0]]))
            Y.append(foot - E.BASE_FOOT[leg])
    sol = np.linalg.lstsq(np.array(A), np.array(Y), rcond=None)[0]
    return np.ascontiguousarray(sol[:20].T), np.ascontiguousarray(sol[20])


@pytest.fixture(scope="session")
def etg_shipped():
    """The gait the reference itself ships (ETGRL/gait_action_list_ETG_exp.npy, 600 samples of info['ETG_act'], sample k = t 0.026(k+1)),
    fitted back to W,b: it walks forward at ~0.48 m/s open loop in the oracle — the long-horizon parity workload."""
    return fit_etg_from_table(np.load(os.path.join(GOLDEN, "gait_action_list_ETG_exp.npy")), 0.026)


def draw_feature_combo(rng):
    """A random combination of the env's feature switches (+ an optional rough height field) for the randomised parity tests."""
    kw = dict(sensor_dis=int(rng.integers(0, 2)), sensor_contact=int(rng.integers(0, 2)), sensor_imu=int(rng.integers(0, 3)), sensor_motor=int(rng.integers(0, 3)),
              sensor_etg=int(rng.integers(0, 2)), obs_normal=int(rng.integers(0, 2)),
              motor_mode=int(rng.choice([0, 0, 1, 2])), joint_limits=int(rng.integers(0, 2)), knee_contacts=int(rng.integers(0, 2)),
              body_collisions=int(rng.integers(0, 2)), stuck_termination=int(rng.integers(0, 2)), external_force=int(rng.integers(0, 2)),
              action_interp=int(rng.integers(0, 2)), action_filter=int(rng.integers(0, 2)), clip_motor_commands=int(rng.integers(0, 2)), max_angle_change=0.2)
    if kw["sensor_dis"] + kw["sensor_contact"] + kw["sensor_imu"] + kw["sensor_motor"] + kw["sensor_etg"] == 0:
        kw["sensor_motor"] = 1
    if rng.integers(0, 2):
        kw["noise_stdev"] = tuple(rng.uniform(0.0, 0.05, 5)); kw["noise_seed"] = int(rng.integers(1, 1000))
    if rng.integers(0, 2):
        kw["base_damping"] = tuple(rng.uniform(0.0, 0.05, 4))
    hf = None
    if rng.integers(0, 2):
        z = rng.uniform(0, 0.03, (40, 40))
        hf = (z, -1.0, -1.0, 0.05)
    return kw, hf
