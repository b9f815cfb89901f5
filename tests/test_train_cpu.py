"""train.py's command line against the reference's ETGRL/train.py:452-505: every flag parses with the reference's default, the options the
batched engine cannot honour raise before any env exists, the argument errors, act_bound, the env configuration of the default flags, and
the cadence of the evaluation block with its e_step sequence.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest
import torch

# the reference's argparse block (train.py:452-505): flag -> default
REFERENCE_FLAGS = {
    "outdir": "train_log", "max_steps": 1e7, "epsilon": 0.4, "gamma": 0.95, "sigma": 0.02, "sigma_decay": 0.99, "popsize": 40, "random_dynamic": 0,
    "random_force": 0, "task_mode": "stairstair", "step_y": 0.05, "load": "", "eval": 0, "render": 0, "suffix": "exp0", "random": 0, "normal": 1,
    "vel_d": 0.5, "ETG_T": 0.5, "reward_p": 5, "footheight": 0.1, "steplen": 0.05, "ETG": 1, "ETG_T2": 0.5, "e_step": 400, "act_mode": "traj",
    "ETG_path": "None", "ETG_H": 20, "stand": 0, "torso": 1.5, "up": 0.6, "tau": 0.07, "feet": 0.3, "badfoot": 0.1, "footcontact": 0.1,
    "act_bound": 0.3, "sensor_dis": 1, "sensor_motor": 1, "sensor_imu": 1, "sensor_contact": 1, "sensor_ETG": 1, "sensor_ETG_obs": 0,
    "sensor_footpose": 0, "sensor_dynamic": 0, "sensor_exforce": 0, "sensor_noise": 0, "timesteps": 5, "timeinterval": 1, "RNN_mode": "None",
    "enable_action_filter": 0, "ES": 1, "es_rpm": 1, "x_noise": 0,
}
# flags this command had before it took the rest of the reference's: their defaults are the batched loop's, kept so that runs stay unchanged
BATCHED_DEFAULTS = {"outdir": "", "max_steps": 400000, "es_rpm": 0}

REFUSED = [["--ETG_H", "16"], ["--ETG_T2", "0.4"], ["--stand", "0.1"], ["--sensor_ETG_obs", "1"], ["--sensor_footpose", "1"], ["--sensor_dynamic", "1"],
           ["--sensor_exforce", "1"], ["--RNN_mode", "GRU"], ["--random_dynamic", "1"], ["--random_force", "1"], ["--x_noise", "1"], ["--render", "1"]]


def _no_device(monkeypatch):
    from paddlerobotics_b200 import train
    fail = lambda *a, **k: pytest.fail("an env was constructed")
    monkeypatch.setattr(train, "VecQuadrupedalEnv", fail)
    monkeypatch.setattr(train, "PopulationEvaluator", fail)
    monkeypatch.setattr(train, "make_envs", fail)
    monkeypatch.setattr(train, "evaluate", fail)
    return train


def test_every_reference_flag_parses_with_the_reference_default():
    from paddlerobotics_b200 import train
    args = vars(train.parser().parse_args([]))
    for k, v in REFERENCE_FLAGS.items():
        assert k in args, k
        assert args[k] == BATCHED_DEFAULTS.get(k, v), (k, args[k], v)
    assert args["train_eval_envs"] == 0 and args["e_step_growth"] == 0        # both new behaviours default off


@pytest.mark.parametrize("extra", REFUSED, ids=lambda e: e[0].lstrip("-"))
def test_refused_flags_raise_before_any_env(monkeypatch, extra):
    train = _no_device(monkeypatch)
    with pytest.raises(NotImplementedError):
        train.main(extra)


def test_ignored_flags_are_accepted(monkeypatch):
    from paddlerobotics_b200 import train
    a = train.parser().parse_args(["--epsilon", "0.1", "--gamma", "0.5", "--random", "1", "--timesteps", "3", "--timeinterval", "2"])
    train.check_supported(a)
    assert train.train_env_config(a).keys() == train.train_env_config(train.parser().parse_args([])).keys()


def test_argument_errors(monkeypatch, tmp_path):
    train = _no_device(monkeypatch)
    with pytest.raises(SystemExit):
        train.main(["--ETG", "0", "--ES", "1"])
    sd = {"actor_model.l1.weight": torch.zeros(256, 49)}
    path = str(tmp_path / "itr_5.pt")
    torch.save(sd, path)
    for extra in ([], ["--eval", "1"]):
        with pytest.raises(SystemExit):
            train.main(["--load", path, "--sensor_dis", "0"] + extra)


def test_act_bound_of_every_mode():
    from paddlerobotics_b200 import bctrain, train
    for mode, want in (("traj", [0.25] * 12), ("pose", [0.1, 0.7, 0.7] * 4), ("torque", [10.0] * 12)):     # train.py:315-320
        a = train.parser().parse_args(["--act_mode", mode, "--act_bound", "0.25"])
        assert np.array_equal(bctrain.act_bound_of(a), np.array(want)), mode
        assert train.train_env_config(a)["motor_mode"] == (1 if mode == "torque" else 0)


def _config(cfg):
    """The B2QConfig VecQuadrupedalEnv builds from these keywords (its __init__'s filling, without a device)."""
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import B2QConfig
    c = B2QConfig()
    _lib.load().b2q_default_config(C.byref(c))
    cfg = dict(cfg)
    field = cfg.pop("heightfield")
    hf = None
    if field is not None:
        hf, x0, y0, cell = field
        c.terrain_type, c.hf_ny, c.hf_nx, c.hf_x0, c.hf_y0, c.hf_cell = 1, hf.shape[0], hf.shape[1], float(x0), float(y0), float(cell)
    for k, v in cfg.items():
        if k in ("noise_stdev", "base_damping"):
            for i, x in enumerate(v):
                getattr(c, k)[i] = float(x)
        else:
            setattr(c, k, v)
    return c, hf


def _fields(c):
    from paddlerobotics_b200._config import B2QConfig
    out = {}
    for name, _ in B2QConfig._fields_:
        if name == "hf_host":
            continue
        v = getattr(c, name)
        out[name] = list(v) if hasattr(v, "__len__") else v
    return out


@pytest.mark.parametrize("task", ["stairstair", "balancebeam", "ground"])
def test_default_flags_give_the_parent_configuration(task):
    from paddlerobotics_b200 import build, train
    from paddlerobotics_b200.terrain import make_terrain
    build.build()
    args = train.parser().parse_args(["--task_mode", task])
    # the parent's train.env_config, written out: the configuration of every training env before this command took the reference's flags
    parent = dict(w_torso=args.torso, w_feet=args.feet, w_up=args.up, w_tau=args.tau, w_badfoot=args.badfoot, w_footcontact=args.footcontact,
                  heightfield=make_terrain(args.task_mode, step_y=args.step_y), stuck_termination=1, body_collisions=1,
                  etg_foot_y_inset=args.step_y if args.task_mode == "balancebeam" else 0.0)
    c_old, hf_old = _config(parent)
    c_new, hf_new = _config(train.train_env_config(args))
    assert _fields(c_old) == _fields(c_new)
    assert (hf_old is None and hf_new is None) or np.array_equal(hf_old, hf_new)


def test_etg_T_reaches_the_env_and_pretrain_config_is_unchanged():
    from paddlerobotics_b200 import pretrain, train
    a = train.parser().parse_args(["--ETG_T", "0.4", "--ETG_T2", "0.4"])
    cfg = train.train_env_config(a)
    assert cfg["etg_T"] == 0.4 and cfg["etg_T2"] == 0.4
    pa = pretrain.parser().parse_args(["--ETG_T", "0.4", "--ETG_T2", "0.4", "--vel_d", "0.6", "--normal", "0"])
    got = pretrain.env_config(pa)
    base = dict(w_torso=pa.torso, w_feet=pa.feet, w_up=pa.up, w_tau=pa.tau, w_badfoot=pa.badfoot, w_footcontact=pa.footcontact, stuck_termination=1,
                body_collisions=1, etg_foot_y_inset=0.0, vel_d=0.6, reward_p=5.0, obs_normal=0, action_filter=0, etg_T=0.4, etg_T2=0.4)
    assert {k: v for k, v in got.items() if k != "heightfield"} == base


def test_sensor_flags_set_the_width_and_noise():
    from paddlerobotics_b200 import train
    a = train.parser().parse_args(["--sensor_dis", "0", "--sensor_noise", "1", "--seed", "7"])
    assert train.obs_width(a) == 46
    cfg = train.train_env_config(a)
    assert cfg["sensor_dis"] == 0 and cfg["noise_seed"] == 7 and len(cfg["noise_stdev"]) == 5


def _reference_blocks(steps_per_episode, num_steps, every, e_step0, growth):
    """train.py:370-385 written out: after each episode of `steps_per_episode` env steps, the evaluations and the e_step growth.  Returns
    [(total_steps, evaluations in the block, e_step after the block)].  test_flag starts at 1 here: the reference's test_flag = 0 also runs a
    block after the very first episode, which the batched loop (whose block is also its checkpoint) does not."""
    EVAL_EVERY_STEPS = every
    total_steps, test_flag, e_step, out = 0, 1, e_step0, []
    while total_steps < num_steps:
        total_steps += steps_per_episode
        if (total_steps + 1) // EVAL_EVERY_STEPS >= test_flag:
            evals = 0
            while (total_steps + 1) // EVAL_EVERY_STEPS >= test_flag:
                test_flag += 1
                evals += 1
            if e_step < 600:
                e_step += growth
            out.append((total_steps, evals, e_step))
    return out


@pytest.mark.parametrize("num_envs", [1, 7, 256, 4096])
def test_block_cadence_and_e_step_sequence_match_the_reference(num_envs):
    """One iteration of the batched loop adds num_envs env steps, as one episode of num_envs steps would in the reference.  With `every` a
    multiple of num_envs of at least two, the blocks also fall where the checkpoints of the earlier `total >= k * every` rule fell."""
    from paddlerobotics_b200 import train
    for every in (int(1e4) * num_envs, 10 * num_envs, 3 * num_envs):
        ref = _reference_blocks(num_envs, 40 * every, every, 400, 50)
        got, total, flag, e_step = [], 0, 1, 400
        while total < 40 * every:
            total += num_envs
            due, flag = train.block_due(total, flag, every)
            if due:
                e_step = train.grow_e_step(e_step, 50)
                got.append((total, 1, e_step))
        assert got == ref, (num_envs, every)
        if num_envs > 1:
            assert [t for t, _, _ in got] == [k * every for k in range(1, 41)]
    assert [train.grow_e_step(e, 50) for e in (400, 550, 600, 650)] == [450, 600, 600, 650]
