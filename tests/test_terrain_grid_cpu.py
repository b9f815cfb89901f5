"""Terrain-grid evaluation without a GPU: terrain_grid enumerates the reference's grids (train.py:48-50) for every task whose terrain uses
them, padded atlas tiles give the heights and normals of their unpadded fields, and every --terrain_grid argument error of train,
pretrain and bctrain is raised before any device work."""
import numpy as np
import pytest
import torch

from paddlerobotics_b200 import terrain

REF_STEP_HEIGHT = np.arange(0.08, 0.101, 0.002)     # train.py:48
REF_SLOPE = np.arange(0.2, 0.401, 0.02)             # train.py:49
REF_STEP_WIDTH = np.arange(0.26, 0.401, 0.02)       # train.py:50
REF = {"step_height": REF_STEP_HEIGHT, "step_width": REF_STEP_WIDTH, "slope": REF_SLOPE}
EXPECTED = {"stairstair": (("step_height", "step_width"), 88), "stairslope": (("step_height", "step_width", "slope"), 968),
            "slopestair": (("step_height", "step_width", "slope"), 968), "slopeslope": (("step_height", "slope"), 121)}


@pytest.mark.parametrize("task", sorted(EXPECTED))
def test_grid_is_the_product_of_the_reference_aranges(task):
    keys, count = EXPECTED[task]
    g = terrain.terrain_grid(task)
    assert len(g) == count and all(tuple(d) == keys for d in g)
    want = set(__import__("itertools").product(*(REF[k].tolist() for k in keys)))
    assert set(tuple(d[k] for k in keys) for d in g) == want and len(want) == count
    for k in keys:                     # the values are the arange's own floats, not re-rounded ones
        assert sorted(set(d[k] for d in g)) == REF[k].tolist()


@pytest.mark.parametrize("task", ["ground", "plane", "balancebeam", "terrain", "nosuchtask"])
def test_tasks_without_a_grid_are_refused(task):
    with pytest.raises(ValueError, match="no terrain grid"):
        terrain.terrain_grid(task)


def _lookup(hf, x0, y0, cell, x, y):
    """terrain_height (b2q_sim.cuh) in float64 NumPy: clamped bilinear height and unit normal."""
    ny, nx = hf.shape
    fx = np.minimum(np.maximum((x - x0) / cell, 0.0), nx - 1.000001)
    fy = np.minimum(np.maximum((y - y0) / cell, 0.0), ny - 1.000001)
    ix, iy = np.minimum(fx.astype(int), nx - 2), np.minimum(fy.astype(int), ny - 2)
    tx, ty = fx - ix, fy - iy
    h00, h10, h01, h11 = hf[iy, ix], hf[iy, ix + 1], hf[iy + 1, ix], hf[iy + 1, ix + 1]
    h = (1 - tx) * (1 - ty) * h00 + tx * (1 - ty) * h10 + (1 - tx) * ty * h01 + tx * ty * h11
    dx = ((1 - ty) * (h10 - h00) + ty * (h11 - h01)) / cell
    dy = ((1 - tx) * (h01 - h00) + tx * (h11 - h10)) / cell
    inv = 1 / np.sqrt(dx * dx + dy * dy + 1)
    return h, -dx * inv, -dy * inv, inv


@pytest.mark.parametrize("task", sorted(EXPECTED))
def test_padded_tiles_equal_make_terrain_and_continue_flat(task):
    g = terrain.terrain_grid(task)
    geoms = [g[0], g[len(g) // 2], g[-1], g[len(g) // 3]]       # both extremes of every grid value among them
    tiles, x0, y0, cell = terrain.make_terrain_tiles(task, geoms)
    assert tiles.dtype == np.float64 and tiles.shape[0] == len(geoms)
    longest = max(terrain.make_terrain(task, **d)[0].shape[1] for d in geoms)
    assert tiles.shape[2] == longest
    for t, d in enumerate(geoms):
        hf, fx0, fy0, fcell = terrain.make_terrain(task, **d)
        assert (fx0, fy0, fcell) == (x0, y0, cell) and tiles.shape[1] == hf.shape[0]
        nx = hf.shape[1]
        assert np.array_equal(tiles[t, :, :nx], hf)                                    # cell by cell inside the field
        assert np.array_equal(tiles[t, :, nx:], np.repeat(hf[:, -1:], longest - nx, 1))  # its last column beyond it
        assert np.all(hf[:, -2:] == 0.0)                                                 # the run-out is flat at the start height
        # the kernel's lookup on both: equal heights and normals everywhere, past the unpadded field's end too
        xs = np.linspace(x0 - 0.5, x0 + cell * (longest - 1) + 0.5, 3001)
        ys = np.linspace(y0 - 0.2, -y0 + 0.2, 7)
        X, Y = np.meshgrid(xs, ys)
        a, b = _lookup(hf, x0, y0, cell, X, Y), _lookup(tiles[t], x0, y0, cell, X, Y)
        for u, v in zip(a, b):
            assert np.array_equal(u, v)


def test_tiles_refuse_an_empty_or_plane_list():
    with pytest.raises(ValueError):
        terrain.make_terrain_tiles("stairstair", [])
    with pytest.raises(ValueError):
        terrain.make_terrain_tiles("ground", [{}])


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
    (["--eval", "1", "LOAD", "--render_dir", "frames"], "--render_dir"),
    (["--eval", "1", "LOAD", "--task_mode", "ground"], "no step height"),
    (["--eval", "1", "LOAD", "--task_mode", "balancebeam"], "no step height"),
]


@pytest.mark.parametrize("command", [_train, _pretrain, _bctrain], ids=["train", "pretrain", "bctrain"])
@pytest.mark.parametrize("extra,message", ERRORS, ids=["no_eval", "render_dir", "ground", "balancebeam"])
def test_argument_errors_come_before_device_work(command, extra, message, monkeypatch, capsys, tmp_path):
    _no_device(monkeypatch)
    argv = ["--terrain_grid", "1"]
    for a in extra:
        argv += ["--load", str(tmp_path / LOADS[command])] if a == "LOAD" else [a]
    with pytest.raises(SystemExit):
        command(argv)
    assert message in capsys.readouterr().err


def test_train_refuses_kernel_sensor_noise(monkeypatch, capsys, tmp_path):
    _no_device(monkeypatch)
    with pytest.raises(SystemExit):
        _train(["--terrain_grid", "1", "--eval", "1", "--load", str(tmp_path / "agent.pt"), "--sensor_noise", "1"])
    assert "--sensor_noise" in capsys.readouterr().err


def test_flag_defaults_off():
    from paddlerobotics_b200 import bctrain, pretrain, train
    for m in (train, pretrain, bctrain):
        assert m.parser().parse_args([]).terrain_grid == 0
