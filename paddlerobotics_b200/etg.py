"""Host-side ETG helpers mirroring the reference's call surface.

ETG_layer / ETG_model live in rlschool (absent from the reference tree); this restatement reproduces the
reference's golden tables gait_action_list_ETG_exp.npy and gait_action_list_CPG_stairstair7_12_3.npy through the
in-tree IK to <=1.3e-14 (SURVEY.md App. A; tests/test_oracle_golden.py).  LS_sol / Opt_with_points /
param2dynamic_dict follow ETGRL/train.py:59-126 (same names, argument meaning and iteration limits) — these run on
the host once per ES individual, not per step; the per-step ETG evaluation itself is inside the CUDA step kernel.
"""
from copy import copy

import numpy as np

POSE_ORI = np.array([0, 0.9, -1.8] * 4)
BASE_FOOT = np.array([[0.18, -0.15, -0.23], [0.18, 0.148, -0.23], [-0.18, -0.14, -0.23], [-0.18, 0.135, -0.23]])
COM_OFFSET = -np.array([0.012731, 0.002186, 0.000515])                      # a1.py:70
HIP_OFFSETS = np.array([[0.183, -0.047, 0.], [0.183, 0.047, 0.], [-0.183, -0.047, 0.], [-0.183, 0.047, 0.]]) + COM_OFFSET  # a1.py:71-73


class ETG_layer:
    """RBF phase features of the ETG (constructor args as ETGRL/train.py:296-297)."""

    def __init__(self, T, dt, H, sigma_sq, phase, amp, T2_radio):
        self.T, self.dt, self.H, self.sigma_sq, self.amp, self.T2 = T, dt, H, sigma_sq, amp, T2_radio
        self.phase = np.asarray(phase, dtype=np.float64)
        self.omega = 2.0 * np.pi / T
        self.u = np.array([self.forward(h * T / (H - 0.9)) for h in range(H)])  # note the H-0.9 denominator
        self.TD = 0

    def forward(self, t):
        return self.amp * np.sin(self.phase + self.omega * t)

    def update(self, t=None):
        x = self.forward(self.TD if t is None else t)
        self.TD += self.dt
        d = x[None, :] - self.u
        return np.exp(-np.sum(d * d, axis=1) / self.sigma_sq)

    def update2(self, t=None, info=None):
        time = self.TD if t is None else t
        self.TD += self.dt
        out = []
        for tt in (time, time + 0.5 * self.T2):
            d = self.forward(tt)[None, :] - self.u
            out.append(np.exp(-np.sum(d * d, axis=1) / self.sigma_sq))
        return out

    def reset(self):
        self.TD = 0


def foot_position_in_hip_frame_to_joint_angle(foot_position, l_hip_sign=1):
    """Closed-form A1 leg IK, same formula as a1.py:97-110 (host copy for table generation / tests)."""
    l_up, l_low, l_hip = 0.2, 0.2, 0.08505 * l_hip_sign
    x, y, z = foot_position
    with np.errstate(invalid="ignore"):
        tk = -np.arccos((x * x + y * y + z * z - l_hip ** 2 - l_low ** 2 - l_up ** 2) / (2 * l_low * l_up))
        l = np.sqrt(l_up ** 2 + l_low ** 2 + 2 * l_up * l_low * np.cos(tk))
        th = np.arcsin(-x / l) - tk / 2
    c1 = l_hip * y - l * np.cos(th + tk / 2) * z
    s1 = l * np.cos(th + tk / 2) * y + l_hip * z
    return np.array([np.arctan2(s1, c1), th, tk])


def foot_position_in_hip_frame(angles, l_hip_sign=1):
    """Closed-form A1 leg FK, same formula as a1.py:113-129 (host copy used to turn a gait table back into ETG weights)."""
    ab, hip, knee = angles
    l_up, l_low, l_hip = 0.2, 0.2, 0.08505 * l_hip_sign
    ld = np.sqrt(l_up ** 2 + l_low ** 2 + 2 * l_up * l_low * np.cos(knee))
    eff = hip + knee / 2
    ox, oz = -ld * np.sin(eff), -ld * np.cos(eff)
    return np.array([ox, np.cos(ab) * l_hip - np.sin(ab) * oz, np.sin(ab) * l_hip + np.cos(ab) * oz])


def fit_etg_from_table(table, t0=0.026, T=0.5, dt=0.026, H=20, sigma_sq=0.04, amp=0.2, phase=(-np.pi / 2, 0.0)):
    """Recover (w [3,20], b [3]) from an info['ETG_act'] table (e.g. the reference's gait_action_list_ETG_exp.npy, whose sample k is
    t = 0.026 (k + 1); deployment tables start at t0 = 0): joint offsets -> feet through the FK -> least squares on the RBF features."""
    layer = ETG_layer(T, dt, H, sigma_sq, np.asarray(phase), amp, T)
    table = np.asarray(table, dtype=np.float64)
    A, Y = [], []
    for k in range(table.shape[0]):
        q = table[k] + POSE_ORI
        for leg in (0, 1):
            foot = foot_position_in_hip_frame(q[3 * leg:3 * leg + 3], (-1) ** (leg + 1)) + HIP_OFFSETS[leg]
            tt = t0 + dt * k + (0.0 if leg == 0 else 0.5 * T)
            A.append(np.concatenate([layer.update(tt), [1.0]]))
            Y.append(foot - BASE_FOOT[leg])
    sol = np.linalg.lstsq(np.array(A), np.array(Y), rcond=None)[0]
    return np.ascontiguousarray(sol[:H].T), np.ascontiguousarray(sol[H])


def shipped_gait():
    """(w, b) of the walking gait the reference ships as ETGRL/gait_action_list_ETG_exp.npy (fitted once by scripts/make_shipped_gait.py
    into data/etg_shipped_gait.npz): ~0.48 m/s open loop on flat ground."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "etg_shipped_gait.npz"))
    return z["w"], z["b"]


class ETG_model:
    """forward(): foot-space deltas per leg (FR,RL in phase; FL,RR half a period later); act_clip(): IK to joint
    offsets relative to POSE_ORI with the shrink-until-finite loop."""

    def __init__(self, task_mode="normal", act_mode="traj", step_y=0.05):
        self.task_mode, self.act_mode, self.step_y = task_mode, act_mode, step_y
        self.pose_ori = POSE_ORI.copy()
        self.base_foot = BASE_FOOT.copy()

    def forward(self, w, b, x):
        a1 = np.asarray(w).dot(np.asarray(x[0]).reshape(-1, 1)).reshape(-1) + b
        a2 = np.asarray(w).dot(np.asarray(x[1]).reshape(-1, 1)).reshape(-1) + b
        out = np.zeros(12)
        if self.task_mode == "gallop":
            out[0:3], out[3:6], out[6:9], out[9:12] = a1, a1, a2, a2
        else:
            out[0:3], out[3:6], out[6:9], out[9:12] = a1, a2, a2, a1
        return out

    def act_clip(self, new_act, robot=None):
        out = np.zeros(12)
        for i in range(4):
            delta = np.array(new_act[3 * i:3 * i + 3], dtype=np.float64)
            for _ in range(200):
                ang = foot_position_in_hip_frame_to_joint_angle(delta + self.base_foot[i] - HIP_OFFSETS[i], (-1) ** (i + 1))
                if not np.isnan(ang).any():
                    break
                delta *= 0.95
            out[3 * i:3 * i + 3] = ang
        return out - self.pose_ori


def etg_act_table(w, b, steps, T=0.5, dt=0.026, H=20, sigma_sq=0.04, amp=0.2, phase=(-np.pi / 2, 0.0), T2=0.5, t0=0.0):
    """info['ETG_act'] for `steps` consecutive control steps (the table env_test.py:43-58 dumps)."""
    layer, model = ETG_layer(T, dt, H, sigma_sq, np.asarray(phase), amp, T2), ETG_model()
    return np.array([model.act_clip(model.forward(w, b, layer.update2(t=t0 + dt * k))) for k in range(steps)])


def LS_sol(A, b, precision=1e-4, alpha=0.05, lamb=1, w0=None):
    """Gradient-descent least squares, ETGRL/train.py:59-79."""
    n, m = A.shape
    x = copy(w0) if w0 is not None else np.zeros((m, 1))
    err = A.dot(x) - b
    err = err.transpose().dot(err)
    i = 0
    while err > precision and i < 1000:
        A1 = A.transpose().dot(A)
        dx = A1.dot(x) - A.transpose().dot(b)
        if w0 is not None:
            dx += lamb * (x - w0)
        x = x - alpha * dx
        err = A.dot(x) - b
        err = err.transpose().dot(err)
        i += 1
    return x


def Opt_with_points(ETG, ETG_T=0.4, points=None, b0=None, w0=None, precision=1e-4, lamb=0.5, plot=False, **kwargs):
    """Fit ETG weights to 6 foot-trajectory control points, ETGRL/train.py:81-110."""
    ts = [0.5 * ETG_T + 0.1, 0, 0.05, 0.1, 0.15, 0.2]
    if points is None:
        Steplength = kwargs.get("Steplength", 0.05)
        Footheight = kwargs.get("Footheight", 0.08)
        Penetration = kwargs.get("Penetration", 0.01)
        points = np.array([[0, -Penetration], [-Steplength, -Penetration * 0.5], [-Steplength * 1.5, 0.6 * Footheight], [0, Footheight],
                           [Steplength * 1.5, 0.6 * Footheight], [Steplength, -Penetration * 0.5]])
    obs = np.array([ETG.update(t) for t in ts]).reshape(-1, 20)
    b = np.mean(points, axis=0) if b0 is None else np.array([b0[0], b0[-1]])
    points_t = points - b
    if w0 is None:
        x1 = LS_sol(A=obs, b=points_t[:, 0].reshape(-1, 1), precision=precision, alpha=0.05)
        x2 = LS_sol(A=obs, b=points_t[:, 1].reshape(-1, 1), precision=precision, alpha=0.05)
    else:
        x1 = LS_sol(A=obs, b=points_t[:, 0].reshape(-1, 1), precision=precision, alpha=0.05, lamb=lamb, w0=w0[0, :].reshape(-1, 1))
        x2 = LS_sol(A=obs, b=points_t[:, 1].reshape(-1, 1), precision=precision, alpha=0.05, lamb=lamb, w0=w0[-1, :].reshape(-1, 1))
    w_ = np.stack((x1, np.zeros((20, 1)), x2), axis=0).reshape(3, -1)
    b_ = np.array([b[0], 0, b[1]])
    return w_, b_, points


def param2dynamic_dict(params):
    """48-vector in [-1,1] -> dynamics dict, ETGRL/train.py:112-126 (same keys and clipping)."""
    param = np.clip(copy(params), -1, 1)
    d = {}
    d["control_latency"] = np.clip(40 + 10 * param[0], 0, 80)
    d["footfriction"] = np.clip(0.2 + 10 * param[1], 0, 20)
    d["basemass"] = np.clip(1.5 + 1 * param[2], 0.5, 3)
    d["baseinertia"] = np.clip(np.ones(3) + 1 * param[3:6], np.array([0.1] * 3), np.array([3] * 3))
    d["legmass"] = np.clip(np.ones(3) + 1 * param[6:9], np.array([0.1] * 3), np.array([3] * 3))
    d["leginertia"] = np.clip(np.ones(12) + 1 * param[9:21], np.array([0.1] * 12), np.array([3] * 12))
    d["motor_kp"] = np.clip(80 * np.ones(12) + 40 * param[21:33], np.array([20] * 12), np.array([200] * 12))
    d["motor_kd"] = np.clip(np.array([1., 2., 2.] * 4) + param[33:45] * np.array([1, 2, 2] * 4), np.array([0] * 12), np.array([5] * 12))
    if param.shape[0] > 45:
        d["gravity"] = np.clip(np.array([0, 0, -10]) + param[45:48] * np.array([2, 2, 10]), np.array([-5, -5, -20]), np.array([5, 5, -4]))
    return d


def dynamic_dict_to_row(d=None, latency_unit_s=1e-3):
    """dynamics dict (param2dynamic_dict keys) -> the engine's 48-column row (B2Q_DYN_DIM layout).
    control_latency is taken in milliseconds (rlschool convention [EXT]); masses/inertias are multipliers."""
    row = np.zeros(48)
    row[0:12] = 100.0
    row[12:24] = np.array([1., 2., 2.] * 4)
    row[24], row[25], row[26:29], row[29:48] = 1.0, 0.002, (0, 0, -10.0), 1.0
    if d:
        if "motor_kp" in d: row[0:12] = d["motor_kp"]
        if "motor_kd" in d: row[12:24] = d["motor_kd"]
        if "footfriction" in d: row[24] = d["footfriction"]
        if "control_latency" in d: row[25] = float(d["control_latency"]) * latency_unit_s
        if "gravity" in d: row[26:29] = d["gravity"]
        if "basemass" in d: row[29] = d["basemass"]
        if "baseinertia" in d: row[30:33] = d["baseinertia"]
        if "legmass" in d: row[33:36] = d["legmass"]
        if "leginertia" in d: row[36:48] = d["leginertia"]
    return row


def param2dynamic_rows(params):
    """[P,48] vectors in [-1,1] -> [P,48] engine rows: dynamic_dict_to_row(param2dynamic_dict(p)) for every p at once, with the same
    elementwise operations in the same order, so every row is bit-identical to the per-vector one."""
    p = np.clip(np.asarray(params, dtype=np.float64).reshape(-1, 48), -1, 1)
    kd0 = np.array([1., 2., 2.] * 4)
    rows = np.empty((p.shape[0], 48))
    rows[:, 0:12] = np.clip(80 * np.ones(12) + 40 * p[:, 21:33], 20, 200)
    rows[:, 12:24] = np.clip(kd0 + p[:, 33:45] * np.array([1, 2, 2] * 4), 0, 5)
    rows[:, 24] = np.clip(0.2 + 10 * p[:, 1], 0, 20)
    rows[:, 25] = np.clip(40 + 10 * p[:, 0], 0, 80) * 1e-3
    rows[:, 26:29] = np.clip(np.array([0, 0, -10]) + p[:, 45:48] * np.array([2, 2, 10]), np.array([-5, -5, -20]), np.array([5, 5, -4]))
    rows[:, 29] = np.clip(1.5 + 1 * p[:, 2], 0.5, 3)
    rows[:, 30:33] = np.clip(np.ones(3) + 1 * p[:, 3:6], 0.1, 3)
    rows[:, 33:36] = np.clip(np.ones(3) + 1 * p[:, 6:9], 0.1, 3)
    rows[:, 36:48] = np.clip(np.ones(12) + 1 * p[:, 9:21], 0.1, 3)
    return rows
