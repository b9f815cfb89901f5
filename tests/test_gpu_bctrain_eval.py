"""bctrain's evaluations on the shared episode loop (train.run_evaluate_episodes): `--eval 1` and random_eval give the records of the loop
they replaced, bit for bit, with one fused statistics launch per control step and no b2q_es_accumulate launch."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
STUDENT = os.path.join(HERE, "golden", "StairStair3_BC1_itr_500383.pt")
GAIT = os.path.join(os.path.dirname(HERE), "paddlerobotics_b200", "data", "etg_shipped_gait.npz")


def _old_run_episodes(env, policy, w, b, act_bound, max_step, x_noise=0):
    """bctrain's evaluation loop before it moved to the shared one: per-term copies of `alive`, 1 + 6 b2q_es_accumulate launches per step."""
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import INFO
    from paddlerobotics_b200.train import EVAL_TERMS
    lib, dev, n, es, stream = _lib.load(), env.device, env.num_envs, env.obs.element_size(), env._stream()
    nt = len(EVAL_TERMS)
    cols = torch.tensor([INFO[k] for k in EVAL_TERMS], device=dev)
    alive = torch.ones(n, dtype=torch.uint8, device=dev)
    ret, length = torch.zeros(n, dtype=env.dtype, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    t_alive, t_sum, t_len = torch.empty(nt, n, dtype=torch.uint8, device=dev), torch.zeros(nt, n, dtype=env.dtype, device=dev), torch.zeros(nt, n, dtype=torch.int32, device=dev)
    t_val = torch.empty(nt, n, dtype=env.dtype, device=dev)
    xo = np.random.uniform(-0.1, 0.1, n) if x_noise else None
    obs = env.reset(w, b, x_offset=xo)
    for steps in range(1, max_step + 2):
        obs, rew, done, info = env.step(policy(obs, steps) * act_bound, donef=steps > max_step)
        t_val.copy_(info.index_select(1, cols).T)
        t_alive.copy_(alive.expand(nt, n))
        for j in range(nt):
            assert lib.b2q_es_accumulate(t_val[j].data_ptr(), done.data_ptr(), t_alive[j].data_ptr(), t_sum[j].data_ptr(), t_len[j].data_ptr(), n, es, stream) == 0
        assert lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), alive.data_ptr(), ret.data_ptr(), length.data_ptr(), n, es, stream) == 0
        if not bool(alive.any()):
            break
    return {"mean_return": float(ret.double().mean()), "mean_length": float(length.double().mean()),
            "terms": {k: float(t_sum[j].double().mean()) for j, k in enumerate(EVAL_TERMS)}}


def _old_eval(argv):
    """bctrain --eval 1 before the shared loop: main's seeding and set-up, then the old loop (which drew --x_noise right before its reset)."""
    import torch
    from paddlerobotics_b200 import bc, bctrain
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import etg_of_path
    args = bctrain.parser().parse_args(argv)
    torch.manual_seed(args.seed); np.random.seed(args.seed)
    w, b = etg_of_path(args.ETG_path, args.ETG_T)
    bound = torch.as_tensor(bctrain.act_bound_of(args), dtype=torch.float32, device="cuda")
    student = MujocoAgent(46, 12, seed=args.seed)
    student.restore(args.load)
    env = bctrain.make_vec_env(args, args.eval_envs, auto_reset=False)
    obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)
    rec = _old_run_episodes(env, lambda o, s: student.predict_batch(obs_mem.observe(o, s, noise=bool(args.sensor_noise), append=False, seed=args.seed)),
                            w, b, bound, bctrain.EVAL_STEPS, x_noise=args.x_noise)
    env.close()
    return {"eval_envs": args.eval_envs, **rec}


@pytest.fixture
def launches(monkeypatch):
    """Counts, from here on, the env steps, the EpisodeStats.step calls and the b2q_es_accumulate launches."""
    from paddlerobotics_b200 import _lib, es
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    lib, n = _lib.load(), {"env_step": 0, "stats_step": 0, "es_accumulate": 0}

    def counted(key, fn):
        def call(*a, **k):
            n[key] += 1
            return fn(*a, **k)
        return call
    monkeypatch.setattr(VecQuadrupedalEnv, "step", counted("env_step", VecQuadrupedalEnv.step))
    monkeypatch.setattr(es.EpisodeStats, "step", counted("stats_step", es.EpisodeStats.step))
    monkeypatch.setattr(lib, "b2q_es_accumulate", counted("es_accumulate", lib.b2q_es_accumulate))
    return n


def _one_launch_per_step(n):
    assert n["env_step"] > 0 and n["stats_step"] == n["env_step"] and n["es_accumulate"] == 0, n


@pytest.mark.parametrize("task", ["stairstair", "ground"])
@pytest.mark.parametrize("x_noise", [[], ["--x_noise", "1", "--seed", "3"]], ids=["x_noise0", "x_noise1_seed3"])
def test_eval_equals_the_old_loop(task, x_noise, launches):
    from paddlerobotics_b200 import bctrain
    argv = ["--eval", "1", "--load", STUDENT, "--ETG_path", GAIT, "--task_mode", task, "--eval_envs", "16", "--sensor_noise", "1"] + x_noise
    rec = bctrain.main(argv)
    _one_launch_per_step(dict(launches))
    assert rec == _old_eval(argv)
    assert set(rec) == {"eval_envs", "mean_return", "mean_length", "terms"}


@pytest.mark.parametrize("task", ["stairstair", "ground"])
def test_random_eval_equals_the_old_loop(task, launches):
    import torch
    from paddlerobotics_b200 import bc, bctrain
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    from paddlerobotics_b200.env import etg_of_path
    args = bctrain.parser().parse_args(["--task_mode", task, "--eval_envs", "16", "--sensor_noise", "1", "--seed", "2"])
    w, b = etg_of_path(GAIT, args.ETG_T)
    bound = torch.as_tensor(bctrain.act_bound_of(args), dtype=torch.float32, device="cuda")
    student = MujocoAgent(46, 12, seed=args.seed)
    student.restore(STUDENT)
    learner = SACLearner(student, args.batch, actor_lr=bctrain.ACTOR_LR, critic_lr=bctrain.CRITIC_LR)
    expert = MujocoAgent(49, 12, seed=1)
    env = bctrain.make_vec_env(args, args.eval_envs, auto_reset=False)
    rec = bctrain.random_eval(args, learner, expert, env, w, b, bound)
    _one_launch_per_step(dict(launches))
    obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)
    stu = _old_run_episodes(env, lambda o, s: learner.actor.forward(obs_mem.observe(o, 1 << 30 | s, noise=True, append=False, seed=args.seed), mode=0)[0][0],
                            w, b, bound, bctrain.RANDOM_EVAL_STEPS)
    ref = _old_run_episodes(env, lambda o, s: expert.predict_batch(o), w, b, bound, bctrain.RANDOM_EVAL_STEPS)
    env.close()
    assert rec == {"eval_return": stu["mean_return"], "eval_length": stu["mean_length"], "ref_return": ref["mean_return"],
                   "ref_length": ref["mean_length"], "ref_ratio": stu["mean_return"] / ref["mean_return"] if ref["mean_return"] != 0 else None,
                   "terms": stu["terms"]}
