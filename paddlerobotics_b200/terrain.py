"""Terrain presets for `make_env(task=...)` as height fields for the engine's bilinear height-field contact.

The reference builds its tasks inside rlschool (absent from the tree; terrains are box collision shapes there, SURVEY
App. B.1).  What the reference tree itself fixes is the task vocabulary and the parameter ranges
(ETGRL/train.py:48-50,462-463):

    STEP_HEIGHT = 0.08 .. 0.10 m     SLOPE = 0.2 .. 0.4     STEP_WIDTH = 0.26 .. 0.40 m     --task_mode stairstair (default)

so the presets below are this repo's own geometry built from exactly those parameters: an approach flat, an ascent
(stairs or ramp), a top platform, a descent (stairs or ramp) and a run-out flat.  Box edges become one-cell-wide
(`cell`, default 0.02 m) ramps under the bilinear interpolation.  Every preset returns `(hf[ny, nx], x0, y0, cell)`, the
`heightfield=` argument of VecQuadrupedalEnv / the `hf_*` fields of B2QConfig.
"""
import numpy as np

STEP_HEIGHT = np.arange(0.08, 0.101, 0.002)      # train.py:48
SLOPE = np.arange(0.2, 0.401, 0.02)              # train.py:49
STEP_WIDTH = np.arange(0.26, 0.401, 0.02)        # train.py:50

TASKS = ("ground", "plane", "stairstair", "stairslope", "slopestair", "slopeslope", "balancebeam", "terrain")
_X0, _Y0, _Y1 = -1.0, -1.5, 1.5


def _profile_to_field(xs, h, cell):
    ny = int(round((_Y1 - _Y0) / cell)) + 1
    return np.repeat(np.asarray(h, dtype=np.float64)[None, :], ny, axis=0), _X0, _Y0, cell


def _stairs(xs, x_start, step_height, step_width, n_steps, up=True, h0=0.0):
    """Staircase profile over xs starting at x_start from height h0; returns (h(xs) contribution, x_end, h_end)."""
    k = np.clip(np.floor((xs - x_start) / step_width) + 1, 0, n_steps)
    k = np.where(xs < x_start, 0, k)
    return h0 + (step_height if up else -step_height) * k, x_start + n_steps * step_width, h0 + (step_height if up else -step_height) * n_steps


def _ramp(xs, x_start, slope, rise, up=True, h0=0.0):
    length = rise / slope
    t = np.clip((xs - x_start) / length, 0.0, 1.0)
    return h0 + (rise if up else -rise) * t, x_start + length, h0 + (rise if up else -rise)


def make_terrain(task, step_height=0.08, step_width=0.3, slope=0.3, n_steps=5, approach=0.8, platform=1.0, runout=3.0, cell=0.02, step_y=0.05,
                 seed=0, roughness=0.03):
    """Height field of a reference task name.  `ground` / `plane` return None (analytic plane in the kernel)."""
    if task in ("ground", "plane"):
        return None
    if task not in TASKS:
        raise NotImplementedError("task %r is not provided (have: %s)" % (task, ", ".join(TASKS)))
    rise = step_height * n_steps
    if task == "balancebeam":
        # a beam along +x at the start height with a drop on both sides; the trot's feet are pulled inward by step_y (train.py:463)
        length = approach + platform + runout
        xs = _X0 + cell * np.arange(int(round((length - _X0) / cell)) + 1)
        ny = int(round((_Y1 - _Y0) / cell)) + 1
        ys = _Y0 + cell * np.arange(ny)
        half = 0.15 - step_y + 0.04
        beam = (np.abs(ys)[:, None] <= half) | (xs[None, :] < approach)
        return np.where(beam, 0.0, -0.3).astype(np.float64), _X0, _Y0, cell
    if task == "terrain":
        length = approach + platform + runout
        nx = int(round((length - _X0) / cell)) + 1
        ny = int(round((_Y1 - _Y0) / cell)) + 1
        rng = np.random.default_rng(seed)
        coarse = rng.uniform(-roughness, roughness, (ny // 10 + 2, nx // 10 + 2))
        yi, xi = np.arange(ny) / 10.0, np.arange(nx) / 10.0
        y0i, x0i = yi.astype(int), xi.astype(int)
        ty, tx = (yi - y0i)[:, None], (xi - x0i)[None, :]
        c = lambda a, b: coarse[np.ix_(y0i + a, x0i + b)]
        hf = (1 - ty) * (1 - tx) * c(0, 0) + (1 - ty) * tx * c(0, 1) + ty * (1 - tx) * c(1, 0) + ty * tx * c(1, 1)
        xs = _X0 + cell * np.arange(nx)
        hf = hf * np.clip((xs - approach * 0.5) / (approach * 0.5), 0.0, 1.0)[None, :]      # flat around the start pose
        return hf.astype(np.float64), _X0, _Y0, cell
    first, second = task[:5], task[5:]              # "stair"/"slope" + "stair"/"slope"
    len1 = n_steps * step_width if first == "stair" else rise / slope
    len2 = n_steps * step_width if second == "stair" else rise / slope
    length = approach + len1 + platform + len2 + runout
    xs = _X0 + cell * np.arange(int(round((length - _X0) / cell)) + 1)
    if first == "stair":
        h1, x1, top = _stairs(xs, approach, step_height, step_width, n_steps, True)
    else:
        h1, x1, top = _ramp(xs, approach, slope, rise, True)
    xd = x1 + platform
    if second == "stair":
        h2, _, _ = _stairs(xs, xd, step_height, step_width, n_steps, False, 0.0)
    else:
        h2, _, _ = _ramp(xs, xd, slope, rise, False, 0.0)
    return _profile_to_field(xs, h1 + h2, cell)


# the grid values each task's make_terrain reads: stairs use the height and width, ramps the slope (and the rise, from the height)
GRID_KEYS = {"stairstair": ("step_height", "step_width"), "stairslope": ("step_height", "step_width", "slope"),
             "slopestair": ("step_height", "step_width", "slope"), "slopeslope": ("step_height", "slope")}
_GRID_VALUES = {"step_height": STEP_HEIGHT, "step_width": STEP_WIDTH, "slope": SLOPE}


def terrain_grid(task):
    """Every geometry of the reference's grids (train.py:48-50) that make_terrain(task) distinguishes, as make_terrain keyword dicts in
    row-major order of GRID_KEYS[task]: 88 for stairstair, 968 for stairslope and slopestair, 121 for slopeslope.  Raises ValueError for
    a task without such a grid (ground, plane, balancebeam, terrain)."""
    if task not in GRID_KEYS:
        raise ValueError("task %r has no terrain grid: its terrain does not depend on the step height, width or slope (grids exist for %s)"
                         % (task, ", ".join(GRID_KEYS)))
    keys = GRID_KEYS[task]
    return [dict(zip(keys, (float(v) for v in vals))) for vals in np.stack(np.meshgrid(*(_GRID_VALUES[k] for k in keys), indexing="ij"), -1).reshape(-1, len(keys))]


def make_terrain_tiles(task, geoms, step_y=0.05):
    """The height fields of `geoms` (make_terrain keyword dicts) on one grid: (tiles [T, ny, nx], x0, y0, cell), the arguments of
    VecQuadrupedalEnv.set_terrain_tiles.  The fields share x0, y0, cell and ny and differ in length; each shorter one is padded to the
    longest with copies of its last column.  Every preset ends in a flat run-out and the kernel clamps a lookup at the field's edge, so a
    padded tile gives the heights and normals of its unpadded field wherever the robot can stand."""
    fields = [make_terrain(task, step_y=step_y, **g) for g in geoms]
    if not fields or any(f is None for f in fields):
        raise ValueError("make_terrain_tiles needs at least one geometry of a height-field task, got %d for %r" % (len(fields), task))
    _, x0, y0, cell = fields[0]
    nx = max(f[0].shape[1] for f in fields)
    tiles = np.empty((len(fields), fields[0][0].shape[0], nx), dtype=np.float64)
    for t, (hf, fx0, fy0, fcell) in enumerate(fields):
        assert (fx0, fy0, fcell, hf.shape[0]) == (x0, y0, cell, tiles.shape[1])
        tiles[t, :, :hf.shape[1]] = hf
        tiles[t, :, hf.shape[1]:] = hf[:, -1:]
    return tiles, x0, y0, cell


def sample_terrain_params(rng):
    """One draw of the reference's per-run terrain parameters (train.py:48-50)."""
    return dict(step_height=float(rng.choice(STEP_HEIGHT)), slope=float(rng.choice(SLOPE)), step_width=float(rng.choice(STEP_WIDTH)))
