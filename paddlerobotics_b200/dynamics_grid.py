"""The dynamics sweep of `--eval 1 --dynamics_grid 1` (train, pretrain, bctrain) and of dynamic_train's identification landscape: each
group of param2dynamic_dict's 48-vector (ETGRL/train.py:112-126) set alone to nine levels that span the support of the reference's
random_dynamic draw, param2dynamic_dict(U(-1, 1)^48).

Settings: 0 is the centre, the run's own dynamics; then group-major, level-minor, 1 + 9 x 9 = 82.  A swept engine row is the run's row
(nominal, or --dynamic_param's) with the group's columns taken from param2dynamic_rows at the level.  Each group's columns depend on that
group's entries alone, so with a --dynamic_param vector P the swept row is param2dynamic_rows(P with the group set to the level), bit
for bit.  Several groups do not bracket the nominal row (latency runs 30-50 ms against the nominal 2 ms, friction is 0 for every level
<= -0.02): that is the reference's space, and every record carries the group's engine values at its level.
"""
import math

import numpy as np

from .etg import param2dynamic_rows

# group -> (its entries of the 48-vector, its columns of the engine row (etg.dynamic_dict_to_row))
GROUPS = {
    "control_latency": (slice(0, 1), slice(25, 26)),
    "footfriction": (slice(1, 2), slice(24, 25)),
    "basemass": (slice(2, 3), slice(29, 30)),
    "baseinertia": (slice(3, 6), slice(30, 33)),
    "legmass": (slice(6, 9), slice(33, 36)),
    "leginertia": (slice(9, 21), slice(36, 48)),
    "motor_kp": (slice(21, 33), slice(0, 12)),
    "motor_kd": (slice(33, 45), slice(12, 24)),
    "gravity": (slice(45, 48), slice(26, 29)),
}
LEVELS = (-1.0, -0.75, -0.5, -0.25, 0.0, 0.25, 0.5, 0.75, 1.0)
CENTRE = "centre"

HELP = ("--eval 1: score on every group of the 48 dynamics parameters (control_latency, footfriction, basemass, baseinertia, legmass, "
        "leginertia, motor_kp, motor_kd, gravity), each set alone to -1, -0.75, ..., 1 of param2dynamic_dict on top of the run's dynamics, "
        "in one batched rollout of --eval_envs envs per setting; one JSON line per setting and a summary")


def settings():
    """[(group, level)] in setting order: (CENTRE, None), then every group at every level."""
    return [(CENTRE, None)] + [(g, l) for g in GROUPS for l in LEVELS]


def _level_rows():
    """{level: the engine row of the 48-vector with every entry at that level}: its columns of a group are that group's at the level."""
    return dict(zip(LEVELS, param2dynamic_rows(np.repeat(np.array(LEVELS)[:, None], 48, 1))))


def swept_rows(row):
    """[82, 48] engine rows, one per setting: `row` (the run's [48] engine row) with the swept group's columns at the level."""
    out = np.repeat(np.asarray(row, dtype=np.float64).reshape(1, 48), len(settings()), 0)
    level_rows = _level_rows()
    for s, (g, l) in enumerate(settings()[1:], 1):
        cols = GROUPS[g][1]
        out[s, cols] = level_rows[l][cols]
    return out


def swept_params(param):
    """[82, 48] 48-vectors, one per setting: `param` with the swept group's entries set to the level (dynamic_train's landscape)."""
    out = np.repeat(np.asarray(param, dtype=np.float64).reshape(1, 48), len(settings()), 0)
    for s, (g, l) in enumerate(settings()[1:], 1):
        out[s, GROUPS[g][0]] = l
    return out


def setting_records():
    """The leading fields of each setting's record: group, level and the group's engine values at the level (a list, or a number for a
    one-column group; the latency in seconds).  The centre's record carries the group CENTRE and the level None."""
    level_rows = _level_rows()
    recs = [{"group": CENTRE, "level": None}]
    for g, l in settings()[1:]:
        v = level_rows[l][GROUPS[g][1]].tolist()
        recs.append({"group": g, "level": l, g: v[0] if len(v) == 1 else v})
    return recs


def _rank(v):
    """A NaN value (a setting whose robot diverged) ranks below every number."""
    return -math.inf if math.isnan(v) else v


def group_summary(recs, key, highest=False):
    """Per group, from the 81 swept records in setting order (the centre's left out): the level with the lowest `key` (the highest with
    highest=True; a NaN ranks lowest), that value, and the range max - min of `key` over the nine levels (NaN when a level's value is
    NaN).  Most sensitive group first: NaN ranges, then by descending range.  -> [{group, worst_level | best_level, worst_<key> |
    best_<key>, range}]."""
    assert len(recs) == len(GROUPS) * len(LEVELS)
    name = "best" if highest else "worst"
    out = []
    for i, g in enumerate(GROUPS):
        rs = recs[i * len(LEVELS):(i + 1) * len(LEVELS)]
        assert all(r["group"] == g for r in rs)
        vals = [float(r[key]) for r in rs]
        pick = (max if highest else min)(range(len(LEVELS)), key=lambda k: _rank(vals[k]))
        span = math.nan if any(math.isnan(v) for v in vals) else max(vals) - min(vals)
        out.append({"group": g, name + "_level": LEVELS[pick], name + "_" + key: vals[pick], "range": span})
    return sorted(out, key=lambda d: (not math.isnan(d["range"]), -d["range"] if not math.isnan(d["range"]) else 0.0))
