"""--eval 1 --dynamics_grid 1 on the GPU: every checked setting's record of train, pretrain and bctrain equals run_evaluate_episodes on a
plain env given that setting's one dynamics row with set_dynamics, compared with ==, in float32 and float64; the centre's record equals
the command's plain --eval 1 record; and dynamic_train's landscape equals --eval 1 --load and one-vector DynamicsEvaluators per vector."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
STUDENT = os.path.join(HERE, "golden", "StairStair3_BC1_itr_500383.pt")
GAIT = os.path.join(os.path.dirname(HERE), "paddlerobotics_b200", "data", "etg_shipped_gait.npz")
STATS = ("mean_return", "mean_length", "success_rate", "terms")


def _gait():
    z = np.load(GAIT)
    return z["w"], z["b"]


def _index(group, level):
    from paddlerobotics_b200.dynamics_grid import settings
    return settings().index((group, level))


# the centre, a latency level, a motor_kp level, and two more groups
PICKS = [0, _index("control_latency", -0.5), _index("motor_kp", 0.5), _index("gravity", -0.5), _index("basemass", 1.0)]


def _same(x, y):
    """== on numbers and nested dicts, with NaN equal to NaN (a diverged setting's record)."""
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(_same(x[k], y[k]) for k in x)
    if isinstance(x, list):
        return len(x) == len(y) and all(_same(u, v) for u, v in zip(x, y))
    return x == y or (isinstance(x, float) and isinstance(y, float) and math.isnan(x) and math.isnan(y))


def _check(recs, run_row, single, picks=PICKS):
    """recs: a dynamics-grid evaluation's records and summary; run_row: the run's [48] engine row; single(row) -> run_evaluate_episodes on
    a plain env with that row."""
    from paddlerobotics_b200 import dynamics_grid as dg
    rows = dg.swept_rows(run_row)
    assert len(recs) == 83
    assert [(r["group"], r["level"]) for r in recs[:-1]] == dg.settings()
    summ = recs[-1]
    assert summ["settings"] == 82 and summ["centre_return"] == recs[0]["mean_return"]
    assert _same(summ["groups"], dg.group_summary(recs[1:-1], "mean_return"))
    for s in picks:
        r = single(rows[s])
        assert _same({k: recs[s][k] for k in STATS}, {k: r[k] for k in STATS}), dg.settings()[s]


def _plain_env(cfg, n, row):
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    env = VecQuadrupedalEnv(n, auto_reset=False, **cfg)
    env.set_dynamics(np.repeat(np.asarray(row)[None], n, 0))
    return env


@pytest.fixture(scope="module")
def checkpoint(tmp_path_factory):
    """A seeded train actor with the shipped gait, and a --dynamic_param vector whose legs stay heavy enough to settle."""
    from paddlerobotics_b200.agent import MujocoAgent
    d = tmp_path_factory.mktemp("ckpt")
    agent = MujocoAgent(49, 12, seed=5)
    w, b = _gait()
    agent.save(str(d / "itr_1.pt"))
    np.savez(d / "itr_1.npz", w=w, b=b, param=np.zeros(12))
    p = np.random.default_rng(4).uniform(-0.25, 0.25, 48)
    np.save(d / "dyn.npy", p)
    return str(d / "itr_1.pt"), str(d / "dyn.npy")


def test_train_records_equal_single_dynamics_evaluations(checkpoint):
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import dynamic_param_row
    ckpt, dyn = checkpoint
    argv = ["--eval", "1", "--load", ckpt, "--eval_envs", "3", "--task_mode", "stairstair", "--dynamic_param", dyn]
    recs = train.main(argv + ["--dynamics_grid", "1"])
    args = train.parser().parse_args(argv)
    cfg = train.train_env_config(args)
    agent = MujocoAgent(49, 12, seed=5)
    agent.restore(ckpt)
    w, b = _gait()

    def single(row):
        env = _plain_env(cfg, args.eval_envs, row)
        r = train.run_evaluate_episodes(env, w, b, policy=lambda o, s: agent.predict_batch(o), act_bound=0.3, max_step=train.EVAL_MAX_STEP)
        env.close()
        return r
    _check(recs, dynamic_param_row(dyn), single)
    plain = train.main(argv)
    assert {k: recs[0][k] for k in ("mean_return", "mean_length", "terms")} == {k: plain[k] for k in ("mean_return", "mean_length", "terms")}


def test_train_records_in_float64(checkpoint):
    """The shared evaluator on a float64 env: the actor reads the observations rounded to float32 on both sides."""
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import dynamic_param_row
    ckpt, dyn = checkpoint
    args = train.parser().parse_args(["--eval", "1", "--load", ckpt, "--eval_envs", "2", "--dynamic_param", dyn, "--dynamics_grid", "1"])
    cfg = dict(train.train_env_config(args), precision="f64")
    agent = MujocoAgent(49, 12, seed=5)
    agent.restore(ckpt)
    policy = lambda o, s: agent.predict_batch(o.float()).double()
    w, b = _gait()
    recs = train.evaluate_dynamics_grid(args, cfg, w, b, policy=policy, act_bound=0.3, max_step=train.EVAL_MAX_STEP)

    def single(row):
        env = _plain_env(cfg, args.eval_envs, row)
        assert env.dtype == torch.float64
        r = train.run_evaluate_episodes(env, w, b, policy=policy, act_bound=0.3, max_step=train.EVAL_MAX_STEP)
        env.close()
        return r
    _check(recs, dynamic_param_row(dyn), single)


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_pretrain_records_equal_single_dynamics_evaluations(precision):
    from paddlerobotics_b200 import pretrain, train
    from paddlerobotics_b200.etg import dynamic_dict_to_row
    argv = ["--eval", "1", "--load", GAIT, "--eval_envs", "2", "--task_mode", "stairstair"]
    args = pretrain.parser().parse_args(argv + ["--dynamics_grid", "1"])
    cfg = pretrain.env_config(args)
    w, b = _gait()
    if precision == "f32":
        recs = pretrain.main(argv + ["--dynamics_grid", "1"])
    else:
        cfg = dict(cfg, precision="f64")
        recs = train.evaluate_dynamics_grid(args, cfg, w, b, policy=None, max_step=pretrain.EVAL_MAX_STEP)

    def single(row):
        env = _plain_env(cfg, args.eval_envs, row)
        r = train.run_evaluate_episodes(env, w, b, policy=None, max_step=pretrain.EVAL_MAX_STEP)
        env.close()
        return r
    _check(recs, dynamic_dict_to_row(), single)
    if precision == "f32":
        plain = pretrain.main(argv)
        assert _same({k: recs[0][k] for k in STATS}, {k: plain[k] for k in STATS})


@pytest.mark.parametrize("x_noise", [[], ["--x_noise", "1", "--seed", "3"]], ids=["x_noise0", "x_noise1_seed3"])
def test_bctrain_records_equal_single_dynamics_evaluations(x_noise):
    """The golden student with sensor noise on the FEAT body, 8 envs per setting: each setting fills one warp of the step kernel."""
    from paddlerobotics_b200 import bc, bctrain, train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import etg_of_path
    from paddlerobotics_b200.etg import dynamic_dict_to_row
    argv = ["--eval", "1", "--load", STUDENT, "--ETG_path", GAIT, "--task_mode", "stairstair", "--eval_envs", "8", "--sensor_noise", "1"] + x_noise
    recs = bctrain.main(argv + ["--dynamics_grid", "1"])
    args = bctrain.parser().parse_args(argv)
    w, b = etg_of_path(args.ETG_path, args.ETG_T)
    bound = torch.as_tensor(bctrain.act_bound_of(args), dtype=torch.float32, device="cuda")
    student = MujocoAgent(46, 12, seed=args.seed)
    student.restore(args.load)

    def single(row):
        # bctrain --eval 1 with one dynamics row: main's seeding, then evaluate's draw of the offsets and its noisy student
        np.random.seed(args.seed)
        env = _plain_env(bctrain.env_kwargs(args), args.eval_envs, row)
        obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)
        xo = np.random.uniform(-0.1, 0.1, args.eval_envs) if args.x_noise else None
        r = train.run_evaluate_episodes(env, w, b, policy=lambda o, s: student.predict_batch(obs_mem.observe(o, s, noise=True, append=False, seed=args.seed)),
                                        act_bound=bound, max_step=bctrain.EVAL_STEPS, x_offset=xo)
        env.close()
        return r
    _check(recs, dynamic_dict_to_row(), single)
    plain = bctrain.main(argv)
    assert {k: recs[0][k] for k in ("mean_return", "mean_length", "terms")} == {k: plain[k] for k in ("mean_return", "mean_length", "terms")}


def test_dynamic_train_landscape_equals_single_vector_evaluations(tmp_path, capsys):
    from test_gpu_dynamic_train import P_STAR, planted_data, write_data
    from paddlerobotics_b200 import dynamic_train
    from paddlerobotics_b200 import dynamics_grid as dg
    from paddlerobotics_b200.es import DynamicsEvaluator
    gait, md = planted_data(P_STAR)
    data = write_data(str(tmp_path / "data"), gait, md)
    p = P_STAR + np.random.default_rng(2).uniform(-0.05, 0.05, 48)
    path = str(tmp_path / "p.npy")
    np.save(path, p)
    recs = dynamic_train.main(["--eval", "1", "--load", path, "--dynamics_grid", "1", "--data_dir", data])
    assert len(recs) == 83 and [(r["group"], r["level"]) for r in recs[:-1]] == dg.settings()
    summ = recs[-1]
    assert (summ["centre_eval_reward"], summ["centre_train_reward"]) == (recs[0]["eval_reward"], recs[0]["train_reward"])
    assert summ["groups"] == dg.group_summary(recs[1:-1], "train_reward", highest=True)
    capsys.readouterr()
    vecs = dg.swept_params(p)
    # train_reward: the mean of the exp and ori rewards as DynamicsEvaluator forms it, each table's robot alone in its warp (a one-vector
    # evaluator on ("exp", "ori") puts both robots in one warp, where one can switch the other's contact solve)
    tables = [DynamicsEvaluator(1, gait, md, keys=(k,), **dynamic_train.evaluator_config()) for k in ("exp", "ori")]
    for s in PICKS:
        v = str(tmp_path / ("v%d.npy" % s))
        np.save(v, vecs[s])
        assert recs[s]["eval_reward"] == dynamic_train.main(["--eval", "1", "--load", v, "--data_dir", data])[0]["eval_reward"], dg.settings()[s]
        for ev in tables:
            ev.evaluate(vecs[s][None])
        mean = torch.stack([ev.reward for ev in tables]).reshape(2, 1).mean(0)
        assert bool(torch.isfinite(mean).all()) and recs[s]["train_reward"] == float(mean[0]), dg.settings()[s]
    for ev in tables:
        ev.env.close()
