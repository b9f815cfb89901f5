"""Terrain atlas (b2q_set_terrain_tiles) and the --terrain_grid 1 evaluations on the GPU: env i of an atlas handle computes what a plain
height-field handle built on its tile computes, bit for bit in both precisions; atlas handles refuse snapshots and rendering; and every
per-geometry record of train, pretrain and bctrain --eval 1 --terrain_grid 1 equals run_evaluate_episodes on a single-terrain env."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
STUDENT = os.path.join(HERE, "golden", "StairStair3_BC1_itr_500383.pt")
GAIT = os.path.join(os.path.dirname(HERE), "paddlerobotics_b200", "data", "etg_shipped_gait.npz")


def _gait():
    z = np.load(GAIT)
    return z["w"], z["b"]


def _same_bits(x, y):
    """Bit for bit, NaN payloads included."""
    if x.dtype.is_floating_point:
        x, y = x.view(torch.int64 if x.element_size() == 8 else torch.int32), y.view(torch.int64 if y.element_size() == 8 else torch.int32)
    return torch.equal(x, y)


def _configs():
    """(name, VecQuadrupedalEnv keywords without the height field): train's eval env (the default body) and make_env's (joint limits and
    knee contacts: the FEAT body)."""
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.env import quadrupedal_config
    a = train.parser().parse_args([])
    t = train.train_env_config(a)
    t.pop("heightfield")
    q, _ = quadrupedal_config("stairslope")
    q.pop("heightfield")
    return {"train": t, "make_env": q}


def _geoms():
    """stairslope extremes: both ends of every grid value, and a middle geometry."""
    from paddlerobotics_b200.terrain import terrain_grid
    g = terrain_grid("stairslope")
    pick = lambda h, w, s: next(d for d in g if (d["step_height"], d["step_width"], d["slope"]) == (h, w, s))
    H, W, S = sorted({d["step_height"] for d in g}), sorted({d["step_width"] for d in g}), sorted({d["slope"] for d in g})
    return [pick(H[0], W[0], S[0]), pick(H[-1], W[-1], S[-1]), pick(H[-1], W[0], S[0]), pick(H[0], W[-1], S[-1]), pick(H[5], W[3], S[5])]


@pytest.mark.parametrize("cfg_name", ["train", "make_env"])
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_atlas_env_equals_a_plain_handle_on_its_tile(cfg_name, precision):
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    from paddlerobotics_b200.terrain import make_terrain_tiles
    cfg = _configs()[cfg_name]
    tiles, x0, y0, cell = make_terrain_tiles("stairslope", _geoms())
    rng = np.random.default_rng(7)
    T, steps = tiles.shape[0], 400
    if cfg_name == "train":
        # the default body: an env's result does not depend on the other robots of its warp, so the envs of a tile may sit anywhere
        tile_of_env = np.concatenate([rng.permutation(T), rng.integers(0, T, 37 - T)]).astype(np.int32)   # shuffled, repeated, non-contiguous
        rng.shuffle(tile_of_env)
    else:
        # the FEAT body switches to its general contact solve for a whole warp of 8 robots at once (b2q_sim.cuh, cm.any(need)), in any
        # handle: an env equals the plain-handle env with the same warp mates, so the tiles are assigned per warp
        blocks = np.concatenate([rng.permutation(T), rng.integers(0, T, 2)])
        rng.shuffle(blocks)
        tile_of_env = np.repeat(blocks, 8).astype(np.int32)
    N = len(tile_of_env)
    dyn = np.stack([dynamic_dict_to_row(param2dynamic_dict(rng.uniform(-0.3, 0.3, 48))) for _ in range(N)])   # every env settles finite
    w, b = _gait()
    kw = dict(precision=precision, auto_reset=True, max_episode_steps=120, **cfg)
    atlas = VecQuadrupedalEnv(N, heightfield=(tiles[0], x0, y0, cell), **kw)
    atlas.set_dynamics(dyn)                      # before the tiles: set_terrain_tiles re-settles with each env's dynamics
    atlas.set_terrain_tiles(tiles, tile_of_env)
    plain = []
    for t in range(T):
        idx = np.flatnonzero(tile_of_env == t)
        e = VecQuadrupedalEnv(len(idx), heightfield=(tiles[t], x0, y0, cell), **kw)
        e.set_dynamics(dyn[idx])
        plain.append((torch.as_tensor(idx, device="cuda"), e))
    outs = [atlas.reset(w, b).clone()]
    for _, e in plain:
        outs.append(e.reset(w, b).clone())
    assert bool(torch.isfinite(outs[0]).all())
    for t, (idx, e) in enumerate(plain):
        assert _same_bits(outs[0][idx], outs[1 + t]), "reset obs of tile %d" % t
    gen = torch.Generator(device="cuda").manual_seed(11)
    resets = 0
    for k in range(steps):
        act = (torch.randn(N, 12, device="cuda", generator=gen) * 0.1).to(atlas.dtype)     # the shipped gait plus a seeded residual
        o, r, d, i = atlas.step(act)
        resets += int(d.sum())
        for t, (idx, e) in enumerate(plain):
            po, pr, pd, pi = e.step(act[idx].contiguous())
            assert _same_bits(o[idx], po) and _same_bits(r[idx], pr) and _same_bits(d[idx], pd) and _same_bits(i[idx], pi), \
                "step %d, tile %d (%s, %s)" % (k, t, cfg_name, precision)
    assert resets > 0                            # auto-reset ran
    for _, e in plain:
        e.close()
    atlas.close()


def test_one_tile_atlas_equals_the_height_field_handle():
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.terrain import make_terrain
    hf = make_terrain("stairstair")
    w, b = _gait()
    for precision in ("f32", "f64"):
        kw = dict(precision=precision, auto_reset=True, max_episode_steps=100, **_configs()["train"])
        a, p = VecQuadrupedalEnv(24, heightfield=hf, **kw), VecQuadrupedalEnv(24, heightfield=hf, **kw)
        a.set_terrain_tiles(hf[0][None], np.zeros(24, np.int32))
        assert torch.equal(a.reset(w, b), p.reset(w, b))
        gen = torch.Generator(device="cuda").manual_seed(3)
        for _ in range(250):
            act = (torch.randn(24, 12, device="cuda", generator=gen) * 0.1).to(a.dtype)
            for x, y in zip(a.step(act), p.step(act)):
                assert torch.equal(x, y)
        a.close(); p.close()


def test_atlas_refusals():
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.terrain import make_terrain
    hf = make_terrain("stairstair")
    env = VecQuadrupedalEnv(4, heightfield=hf)
    lib = env.lib
    tile = np.ascontiguousarray(hf[0][None])
    bad = np.array([0, 1, 0, 0], np.int32)
    assert lib.b2q_set_terrain_tiles(env.h, tile.ctypes.data, 1, bad.ctypes.data, None) == -1
    assert b"tile_of_env[1] = 1" in lib.b2q_last_error(env.h)
    assert lib.b2q_set_terrain_tiles(env.h, tile.ctypes.data, 0, np.zeros(4, np.int32).ctypes.data, None) == -1
    assert b"n_tiles" in lib.b2q_last_error(env.h)
    blob = torch.empty(int(lib.b2q_snapshot_bytes(env.h)), dtype=torch.uint8, device="cuda")
    assert lib.b2q_snapshot_save(env.h, blob.data_ptr(), None) == 0             # a plain handle still saves
    env.set_terrain_tiles(tile, np.zeros(4, np.int32))
    for call, what in ((lib.b2q_snapshot_save, b"b2q_snapshot_save"), (lib.b2q_snapshot_load, b"b2q_snapshot_load")):
        assert call(env.h, blob.data_ptr(), None) == -1
        assert what in lib.b2q_last_error(env.h) and b"terrain-atlas" in lib.b2q_last_error(env.h)
    st = env.get_state()
    ids = torch.zeros(1, dtype=torch.int32, device="cuda")
    m = torch.eye(4, device="cuda").reshape(16)
    img = torch.empty(8, 8, 4, dtype=torch.uint8, device="cuda")
    assert lib.b2q_render(env.h, st.data_ptr(), ids.data_ptr(), 1, m.data_ptr(), m.data_ptr(), 8, 8, img.data_ptr(), None, None, None) == -1
    assert b"terrain-atlas" in lib.b2q_last_error(env.h)
    for call in (env.state_dict, lambda: env.load_state_dict({}), lambda: env.get_camera_image(8, 8)):
        with pytest.raises(RuntimeError, match="terrain-atlas"):
            call()
    env.close()
    plane = VecQuadrupedalEnv(2)
    with pytest.raises(ValueError):
        plane.set_terrain_tiles(tile, np.zeros(2, np.int32))
    assert plane.lib.b2q_set_terrain_tiles(plane.h, tile.ctypes.data, 1, np.zeros(2, np.int32).ctypes.data, None) == -1
    assert b"height-field handle" in plane.lib.b2q_last_error(plane.h)
    plane.close()


def _check_geometries(recs, task, single, n_check=4):
    """recs: a grid evaluation's records; single(geom) -> run_evaluate_episodes on a single-terrain env of that geometry."""
    from paddlerobotics_b200.terrain import GRID_KEYS, terrain_grid
    geoms = terrain_grid(task)
    assert len(recs) == len(geoms) + 1 and recs[-1]["geometries"] == len(geoms)
    worst = min(recs[:-1], key=lambda r: r["mean_return"])
    assert recs[-1]["worst_return"] == worst["mean_return"] and recs[-1]["worst"] == {k: worst[k] for k in GRID_KEYS[task]}
    for g in np.linspace(0, len(geoms) - 1, n_check).astype(int):
        rec = recs[g]
        assert {k: rec[k] for k in GRID_KEYS[task]} == geoms[g]
        r = single(geoms[g])
        assert {k: rec[k] for k in ("mean_return", "mean_length", "success_rate", "terms")} == \
            {k: r[k] for k in ("mean_return", "mean_length", "success_rate", "terms")}, geoms[g]


def test_train_grid_records_equal_single_terrain_evaluations(tmp_path):
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.terrain import make_terrain
    agent = MujocoAgent(49, 12, seed=5)
    w, b = _gait()
    agent.save(str(tmp_path / "itr_1.pt"))
    np.savez(tmp_path / "itr_1.npz", w=w, b=b, param=np.zeros(12))
    argv = ["--eval", "1", "--terrain_grid", "1", "--load", str(tmp_path / "itr_1.pt"), "--eval_envs", "3", "--task_mode", "stairstair"]
    recs = train.main(argv)
    args = train.parser().parse_args(argv)
    cfg = train.train_env_config(args)

    def single(geom):
        env = train.make_eval_env(args, dict(cfg, heightfield=make_terrain("stairstair", step_y=args.step_y, **geom)), args.eval_envs)
        r = train.run_evaluate_episodes(env, w, b, policy=lambda o, s: agent.predict_batch(o), act_bound=0.3, max_step=train.EVAL_MAX_STEP)
        env.close()
        return r
    _check_geometries(recs, "stairstair", single)


def test_pretrain_grid_records_equal_single_terrain_evaluations():
    from paddlerobotics_b200 import pretrain, train
    from paddlerobotics_b200.terrain import make_terrain
    argv = ["--eval", "1", "--terrain_grid", "1", "--load", GAIT, "--eval_envs", "2", "--task_mode", "slopeslope"]
    recs = pretrain.main(argv)
    args = pretrain.parser().parse_args(argv)
    cfg = pretrain.env_config(args)
    w, b = _gait()

    def single(geom):
        env = train.make_eval_env(args, dict(cfg, heightfield=make_terrain("slopeslope", step_y=args.step_y, **geom)), args.eval_envs)
        r = train.run_evaluate_episodes(env, w, b, policy=None, max_step=pretrain.EVAL_MAX_STEP)
        env.close()
        return r
    _check_geometries(recs, "slopeslope", single)


@pytest.mark.parametrize("x_noise", [[], ["--x_noise", "1", "--seed", "3"]], ids=["x_noise0", "x_noise1_seed3"])
def test_bctrain_grid_records_equal_single_terrain_evaluations(x_noise):
    from paddlerobotics_b200 import bc, bctrain, train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv, apply_dynamic_param, etg_of_path
    from paddlerobotics_b200.terrain import make_terrain
    argv = ["--eval", "1", "--load", STUDENT, "--ETG_path", GAIT, "--task_mode", "stairstair", "--eval_envs", "16", "--sensor_noise", "1",
            "--terrain_grid", "1"] + x_noise
    recs = bctrain.main(argv)
    args = bctrain.parser().parse_args(argv)
    w, b = etg_of_path(args.ETG_path, args.ETG_T)
    bound = torch.as_tensor(bctrain.act_bound_of(args), dtype=torch.float32, device="cuda")
    student = MujocoAgent(46, 12, seed=args.seed)
    student.restore(args.load)

    def single(geom):
        # bctrain --eval 1 on one geometry: main's seeding, then evaluate's draw of the offsets and its noisy student
        np.random.seed(args.seed)
        cfg = dict(bctrain.env_kwargs(args), heightfield=make_terrain("stairstair", step_y=args.step_y, **geom))
        env = apply_dynamic_param(VecQuadrupedalEnv(args.eval_envs, auto_reset=False, **cfg), args.dynamic_param)
        obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)
        xo = np.random.uniform(-0.1, 0.1, args.eval_envs) if args.x_noise else None
        r = train.run_evaluate_episodes(env, w, b, policy=lambda o, s: student.predict_batch(obs_mem.observe(o, s, noise=True, append=False, seed=args.seed)),
                                        act_bound=bound, max_step=bctrain.EVAL_STEPS, x_offset=xo)
        env.close()
        return r
    _check_geometries(recs, "stairstair", single)
