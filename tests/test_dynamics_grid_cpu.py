"""Dynamics-sweep evaluation without a GPU: the 82 settings and their levels, the swept engine rows against param2dynamic_rows bit for bit
(nominal and with a --dynamic_param vector), dynamic_train's landscape vectors, the per-group summary, and every --dynamics_grid
argument error of train, pretrain, bctrain and dynamic_train raised before any device work."""
import math

import numpy as np
import pytest
import torch

from paddlerobotics_b200 import dynamics_grid as dg
from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict, param2dynamic_rows

GROUPS = ["control_latency", "footfriction", "basemass", "baseinertia", "legmass", "leginertia", "motor_kp", "motor_kd", "gravity"]
SIZES = [1, 1, 1, 3, 3, 12, 12, 12, 3]
LEVELS = [-1.0, -0.75, -0.5, -0.25, 0.0, 0.25, 0.5, 0.75, 1.0]
RNG = np.random.default_rng(11)
P = RNG.uniform(-1, 1, 48)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def test_settings_are_the_centre_then_group_major_level_minor():
    s = dg.settings()
    assert len(s) == 82 and s[0] == (dg.CENTRE, None)
    assert s[1:] == [(g, l) for g in GROUPS for l in LEVELS]
    assert list(dg.GROUPS) == GROUPS and list(dg.LEVELS) == LEVELS
    assert [dg.GROUPS[g][0].stop - dg.GROUPS[g][0].start for g in GROUPS] == SIZES
    assert [dg.GROUPS[g][1].stop - dg.GROUPS[g][1].start for g in GROUPS] == SIZES


def test_groups_partition_the_vector_and_the_row():
    entries = np.concatenate([np.arange(48)[dg.GROUPS[g][0]] for g in GROUPS])
    cols = np.concatenate([np.arange(48)[dg.GROUPS[g][1]] for g in GROUPS])
    assert sorted(entries) == list(range(48)) and sorted(cols) == list(range(48))
    assert list(entries) == list(range(48))                        # param2dynamic_dict's key order is the vector's order


@pytest.mark.parametrize("group", GROUPS)
def test_a_group_s_columns_depend_on_its_entries_alone(group):
    """param2dynamic_rows maps each group's entries to its columns and to nothing else: the premise of the swept-row rule."""
    ent, col = dg.GROUPS[group]
    a = RNG.uniform(-1.5, 1.5, (64, 48))
    b = RNG.uniform(-1.5, 1.5, (64, 48))
    b[:, ent] = a[:, ent]
    ra, rb = param2dynamic_rows(a), param2dynamic_rows(b)
    assert np.array_equal(_bits(ra[:, col]), _bits(rb[:, col]))
    # and the columns are those of the dict's key
    d = param2dynamic_dict(a[0])
    assert np.array_equal(_bits(ra[0, col]), _bits(dynamic_dict_to_row({group: d[group]})[col]))


@pytest.mark.parametrize("with_param", [False, True], ids=["nominal", "dynamic_param"])
def test_swept_rows_equal_param2dynamic_rows_of_the_modified_vector(with_param):
    run_row = dynamic_dict_to_row(param2dynamic_dict(P)) if with_param else dynamic_dict_to_row()
    rows = dg.swept_rows(run_row)
    assert rows.shape == (82, 48) and rows.dtype == np.float64
    assert np.array_equal(_bits(rows[0]), _bits(run_row))                    # the centre is the run's own row
    base = P if with_param else np.zeros(48)
    for s, (g, l) in enumerate(dg.settings()[1:], 1):
        ent, col = dg.GROUPS[g]
        outside = np.ones(48, bool)
        outside[col] = False
        assert np.array_equal(_bits(rows[s][outside]), _bits(run_row[outside])), (g, l)
        q = base.copy()
        q[ent] = l
        want = param2dynamic_rows(q[None])[0]
        if with_param:
            assert np.array_equal(_bits(rows[s]), _bits(want)), (g, l)
        else:
            assert np.array_equal(_bits(rows[s][col]), _bits(want[col])), (g, l)


def test_levels_span_the_reference_space():
    """The record values: latency 30-50 ms in seconds, friction 0 for every level <= -0.02 (so the four lowest levels), kp 40-120."""
    recs = dg.setting_records()
    assert recs[0] == {"group": dg.CENTRE, "level": None}
    rows = dg.swept_rows(dynamic_dict_to_row())
    for s, r in enumerate(recs[1:], 1):
        g, l = dg.settings()[s]
        assert (r["group"], r["level"]) == (g, l) and list(r) == ["group", "level", g]
        v = rows[s][dg.GROUPS[g][1]].tolist()
        assert r[g] == (v[0] if len(v) == 1 else v)
    by = {(r["group"], r["level"]): r for r in recs[1:]}
    assert [by["control_latency", l]["control_latency"] for l in LEVELS] == [0.04 + 0.01 * l for l in LEVELS]
    assert [by["footfriction", l]["footfriction"] for l in LEVELS[:4]] == [0.0] * 4
    assert by["motor_kp", -1.0]["motor_kp"] == [40.0] * 12 and by["motor_kp", 1.0]["motor_kp"] == [120.0] * 12
    assert by["gravity", -1.0]["gravity"] == [-2.0, -2.0, -20.0]


def test_landscape_vectors_equal_the_loaded_vector_outside_the_swept_group():
    v = dg.swept_params(P)
    assert v.shape == (82, 48) and np.array_equal(_bits(v[0]), _bits(P))
    for s, (g, l) in enumerate(dg.settings()[1:], 1):
        ent = dg.GROUPS[g][0]
        outside = np.ones(48, bool)
        outside[ent] = False
        assert np.array_equal(_bits(v[s][outside]), _bits(P[outside])) and np.all(v[s][ent] == l), (g, l)
    # the landscape's engine rows are the commands' swept rows around the same vector
    assert np.array_equal(_bits(param2dynamic_rows(v)), _bits(dg.swept_rows(param2dynamic_rows(P[None])[0])))


def test_dynamic_param_row_is_the_applied_row(tmp_path):
    from paddlerobotics_b200.env import dynamic_param_row
    path = str(tmp_path / "p.npy")
    np.save(path, P)
    assert np.array_equal(_bits(dynamic_param_row(path)), _bits(dynamic_dict_to_row(param2dynamic_dict(P))))
    assert np.array_equal(_bits(dynamic_param_row("")), _bits(dynamic_dict_to_row()))


def _records(values):
    return [{"group": g, "level": l, "v": values.get((g, l), 0.0)} for g, l in dg.settings()[1:]]


def test_group_summary_orders_by_range_and_ranks_nan_lowest():
    vals = {("motor_kp", -1.0): -5.0, ("motor_kp", 1.0): 3.0, ("gravity", 0.5): 1.0, ("legmass", -1.0): math.nan, ("legmass", 1.0): 2.0}
    worst = dg.group_summary(_records(vals), "v")
    assert [d["group"] for d in worst[:3]] == ["legmass", "motor_kp", "gravity"]
    assert [d["group"] for d in worst[3:]] == [g for g in GROUPS if g not in ("legmass", "motor_kp", "gravity")]    # ties keep group order
    assert worst[0]["worst_level"] == -1.0 and math.isnan(worst[0]["worst_v"]) and math.isnan(worst[0]["range"])
    assert worst[1] == {"group": "motor_kp", "worst_level": -1.0, "worst_v": -5.0, "range": 8.0}
    assert worst[2] == {"group": "gravity", "worst_level": -1.0, "worst_v": 0.0, "range": 1.0}      # the first of the tied lowest levels
    best = dg.group_summary(_records(vals), "v", highest=True)
    assert best[1] == {"group": "motor_kp", "best_level": 1.0, "best_v": 3.0, "range": 8.0}
    assert best[0]["best_level"] == 1.0 and best[0]["best_v"] == 2.0


def _no_device(monkeypatch):
    from paddlerobotics_b200 import _lib, env
    fail = lambda *a, **k: pytest.fail("device work before the argument error")
    monkeypatch.setattr(torch.cuda, "_lazy_init", fail)
    monkeypatch.setattr(_lib, "load", fail)
    monkeypatch.setattr(env.VecQuadrupedalEnv, "__init__", fail)


def _train(extra):
    from paddlerobotics_b200 import train
    return train.main(extra)


def _pretrain(extra):
    from paddlerobotics_b200 import pretrain
    return pretrain.main(extra)


def _bctrain(extra):
    from paddlerobotics_b200 import bctrain
    return bctrain.main(extra)


LOADS = {_train: "agent.pt", _pretrain: "gait.npz", _bctrain: "student.pt"}
ERRORS = [
    ([], "needs --eval 1"),
    (["--eval", "1", "LOAD", "--terrain_grid", "1"], "--terrain_grid"),
    (["--eval", "1", "LOAD", "--render_dir", "frames"], "--render_dir"),
]


@pytest.mark.parametrize("command", [_train, _pretrain, _bctrain], ids=["train", "pretrain", "bctrain"])
@pytest.mark.parametrize("extra,message", ERRORS, ids=["no_eval", "terrain_grid", "render_dir"])
def test_argument_errors_come_before_device_work(command, extra, message, monkeypatch, capsys, tmp_path):
    _no_device(monkeypatch)
    argv = ["--dynamics_grid", "1"]
    for a in extra:
        argv += ["--load", str(tmp_path / LOADS[command])] if a == "LOAD" else [a]
    with pytest.raises(SystemExit):
        command(argv)
    err = capsys.readouterr().err
    assert "--dynamics_grid" in err and message in err


def test_train_refuses_kernel_sensor_noise(monkeypatch, capsys, tmp_path):
    _no_device(monkeypatch)
    with pytest.raises(SystemExit):
        _train(["--dynamics_grid", "1", "--eval", "1", "--load", str(tmp_path / "agent.pt"), "--sensor_noise", "1"])
    err = capsys.readouterr().err
    assert "--dynamics_grid" in err and "--sensor_noise" in err


def test_dynamic_train_refuses_a_landscape_without_eval(monkeypatch, capsys, tmp_path):
    from paddlerobotics_b200 import dynamic_train
    _no_device(monkeypatch)
    monkeypatch.setattr(dynamic_train, "load_data", lambda d: pytest.fail("data read before the argument error"))
    with pytest.raises(SystemExit) as e:
        dynamic_train.main(["--dynamics_grid", "1", "--load", str(tmp_path / "p.npy")])
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert "--dynamics_grid" in err and "--eval 1" in err


def test_flag_defaults_off():
    from paddlerobotics_b200 import bctrain, dynamic_train, pretrain, train
    for m in (train, pretrain, bctrain, dynamic_train):
        assert m.parser().parse_args([]).dynamics_grid == 0
