"""The full dynamics-randomisation range: the rows that make_env's random_dynamics and es.DynamicsEvaluator draw, i.e.
param2dynamic_dict over all of [-1, 1]^48, shared by tests/test_emu_full_range.py (CPU emulation) and tests/test_gpu_full_range.py.

Over that range the foot friction runs from 0 to 10.2, the motor kd reaches 0, gravity spans -4 to -20 and tilts by up to +-2, the
link-mass and inertia multipliers reach 0.1 and 3, and the control latency is 30-50 ms (longer than one 26 ms control step).

The row set is 24 seeded draws plus corner rows: one clipped extreme at a time on top of the engine's nominal row.  The float64
oracle classifies every row once: `finite`, or `diverging` when its settle (500 substeps holding the reset pose) already ends
non-finite.  A row is kept only if its class survives a 1e-3 relative perturbation of its mass and inertia multipliers, so no test sits
on the stability boundary.  Rows that diverge have light legs together with light leg inertias; no single clipped extreme diverges on
its own (see DESIGN.md, "Full-range dynamics rows")."""
import functools

import numpy as np

from oracle import oracle as O

SEED, NDRAW = 0, 24
NOMINAL_KD = np.array([1.0, 2.0, 2.0] * 4)
MASS_NAMES = ["basemass"] + ["baseinertia%d" % i for i in range(3)] + ["legmass%d" % i for i in range(3)] + ["leginertia%d" % i for i in range(12)]


def _nominal():
    from paddlerobotics_b200.etg import dynamic_dict_to_row
    return dynamic_dict_to_row()


def _corners():
    """name -> row: each clipped extreme of param2dynamic_dict's domain alone on the nominal row (columns: kp 0-11, kd 12-23, friction 24,
    latency 25 [s], gravity 26-28, base mass 29, base inertia 30-32, leg masses 33-35, leg inertias 36-47)."""
    c = {"fric_0": (24, 0.0), "fric_10.2": (24, 10.2), "kd_0": (slice(12, 24), 0.0), "kd_max": (slice(12, 24), 2.0 * NOMINAL_KD),
         "kp_40": (slice(0, 12), 40.0), "kp_120": (slice(0, 12), 120.0), "g_-4": (28, -4.0), "g_-20": (28, -20.0),
         "gx_+2": (26, 2.0), "gx_-2": (26, -2.0), "gy_+2": (27, 2.0), "gy_-2": (27, -2.0), "lat_30ms": (25, 0.030), "lat_50ms": (25, 0.050)}
    for j, nm in enumerate(MASS_NAMES):
        c[nm + "_0.1"] = (29 + j, 0.1)
        c[nm + "_3"] = (29 + j, 3.0)
    out = {}
    for name, (col, v) in c.items():
        r = _nominal()
        r[col] = v
        out[name] = r
    return out


def drawn_rows():
    """name -> row of the seeded draws param2dynamic_dict(uniform(-1, 1, 48))."""
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    x = np.random.default_rng(SEED).uniform(-1, 1, (NDRAW, 48))
    return {"draw_%02d" % i: dynamic_dict_to_row(param2dynamic_dict(x[i])) for i in range(NDRAW)}


def settles_finite(row):
    o = O.OracleEnv(O.default_config(), row)
    ob = o.reset()
    return bool(np.isfinite(ob).all() and np.isfinite(o.get_state()).all())


def classify(row):
    """"finite", "diverging", or None when a 1e-3 relative change of the mass / inertia multipliers changes the class."""
    c = []
    for f in (1.0, 1.0 + 1e-3, 1.0 - 1e-3):
        r = row.copy()
        r[29:48] *= f
        c.append(settles_finite(r))
    return "finite" if all(c) else "diverging" if not any(c) else None


@functools.lru_cache(maxsize=None)
def row_set():
    """(finite, diverging): name -> row dicts of the classified full-range rows, in a fixed order."""
    rows = dict(drawn_rows(), **_corners())
    fin, div = {}, {}
    for name, r in rows.items():
        c = classify(r)
        if c == "finite":
            fin[name] = r
        elif c == "diverging":
            div[name] = r
    return fin, div


def warmup_steps(latency, dt=0.002, repeat=13):
    """Control steps whose delayed (control-latency) observation still reads the history the reset filled from the settled snapshot.

    The observation of step k interpolates the substep states n_lag and n_lag + 1 before the last substep, n_lag = int(latency / dt);
    that reaches back into step k - ceil((n_lag + 2 - repeat) / repeat).  A teacher-forced comparison loads the oracle's state, not its
    history, so on these steps the two sides read their own (float32 vs float64) settles.  n_lag is taken one larger than float64
    gives, because float32 may round latency / dt up across an integer."""
    if latency <= 0:
        return 0
    n_lag = int(latency / dt) + 1
    return max(0, -(-(n_lag + 2 - repeat) // repeat))


def adopt_reset_orientation(oracles, reset_state):
    """Give every oracle the engine's reset orientation as its heading reference (obs 7-9 are (rpy - rpy0) / 0.1, rpy0 taken at reset).

    rpy0 is per-episode state that teacher forcing does not load.  It comes from the settled snapshot, so without this the two settles'
    difference would stay in obs 7-9 on every step.  The settles themselves are compared on their own, at reset."""
    for o, s in zip(oracles, np.asarray(reset_state, np.float64)):
        rpy = O.quat_to_rpy(s[3:7])
        for k in range(3):
            o.e.rpy0[k] = float(rpy[k])

