"""train, pretrain and bctrain under torchrun, without a GPU: the refusals of a multi-rank run are argument errors (or NotImplementedError)
raised before any device work or process group, and with no rank variables train hands its loop today's configuration, seeds and
learner arguments."""
import numpy as np
import pytest
import torch


def _no_device(monkeypatch):
    import torch.distributed as dist
    from paddlerobotics_b200 import bctrain, dist_run, pretrain, train
    fail = lambda *a, **k: pytest.fail("device work or a process group started")
    for name in ("VecQuadrupedalEnv", "PopulationEvaluator", "make_envs", "evaluate", "run"):
        monkeypatch.setattr(train, name, fail)
    monkeypatch.setattr(pretrain, "pretrain", fail)
    monkeypatch.setattr(pretrain, "evaluate", fail)
    monkeypatch.setattr(bctrain, "MujocoAgent", fail)
    monkeypatch.setattr(dist_run, "process_group", fail)
    monkeypatch.setattr(dist, "init_process_group", fail)
    return train, pretrain, bctrain


@pytest.fixture
def two_ranks(monkeypatch):
    for k, v in (("RANK", "1"), ("WORLD_SIZE", "2"), ("LOCAL_RANK", "1")):
        monkeypatch.setenv(k, v)
    return _no_device(monkeypatch)


@pytest.mark.parametrize("flag", ["num_envs", "batch", "memory", "popsize"])
def test_train_size_not_divisible_by_the_ranks(two_ranks, flag, capsys):
    train = two_ranks[0]
    with pytest.raises(SystemExit):
        train.main(["--graph_iter", "0", "--" + flag, "41"])
    assert "--%s 41 must be divisible by the 2 ranks" % flag in capsys.readouterr().err


def test_train_gloo_with_the_captured_iteration(two_ranks, capsys):
    train = two_ranks[0]
    with pytest.raises(SystemExit):
        train.main(["--dist_backend", "gloo"])                  # --graph_iter 1 is the default
    assert "cannot be captured" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        train.main(["--dist_backend", "mpi", "--graph_iter", "0"])


@pytest.mark.parametrize("extra", [["--save_state", "1", "--outdir", "o"], ["--resume", "o/exp0/state.pt"]], ids=["save_state", "resume"])
def test_train_state_files_are_single_gpu(two_ranks, extra):
    train = two_ranks[0]
    with pytest.raises(NotImplementedError, match="run it on one GPU"):
        train.main(extra)


def test_bctrain_is_single_gpu(two_ranks):
    bctrain = two_ranks[2]
    with pytest.raises(NotImplementedError, match="run it on one GPU"):
        bctrain.main([])


def test_pretrain_popsize_not_divisible_by_the_ranks(two_ranks, capsys):
    pretrain = two_ranks[1]
    with pytest.raises(SystemExit):
        pretrain.main(["--popsize", "41"])
    assert "--popsize 41 must be divisible by the 2 ranks" in capsys.readouterr().err


def test_eval_on_the_other_ranks_returns_at_once(two_ranks, tmp_path):
    train, pretrain, _ = two_ranks
    sd = {"actor_model.l1.weight": torch.zeros(256, 49)}
    torch.save(sd, tmp_path / "itr_5.pt")
    assert train.main(["--eval", "1", "--load", str(tmp_path / "itr_5.pt"), "--graph_iter", "0"]) == []
    assert pretrain.main(["--eval", "1", "--load", "x.npz"]) == []


def test_one_rank_without_a_process_group(monkeypatch):
    import torch.distributed as dist
    from paddlerobotics_b200 import dist_run
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setattr(dist, "init_process_group", lambda *a, **k: pytest.fail("a process group at world 1"))
    assert dist_run.ranks() == (0, 1, 0)
    with dist_run.process_group(1, 0, "nccl") as dev:
        assert dev == 0


class _Stop(Exception):
    pass


def test_one_rank_hands_the_loop_todays_arguments(monkeypatch):
    """No rank variables: the env configuration (sensor noise seeded by --seed), torch's seed, the shard sizes and the learner's arguments
    are the single-GPU ones."""
    from paddlerobotics_b200 import train
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    seeds, seen = [], {}
    monkeypatch.setattr(torch, "manual_seed", lambda s: seeds.append(s))

    class Env:
        observation_dim = 49
    made = {}

    def make_envs(args, env_cfg, policy=None, act_bound=None, rank=0, world=1, device=0):
        made.update(env_cfg=env_cfg, rank=rank, world=world, device=device, n=args.num_envs // world)
        return Env(), None

    def learner(agent, batch, **kw):
        seen.update(batch=batch, **kw)
        raise _Stop
    monkeypatch.setattr(train, "make_envs", make_envs)
    monkeypatch.setattr(train, "MujocoAgent", lambda od, ad, device=0, seed=0: made.update(agent=(od, ad, device, seed)))
    monkeypatch.setattr(train, "SACLearner", learner)
    import torch.distributed as dist
    monkeypatch.setattr(dist, "init_process_group", lambda *a, **k: pytest.fail("a process group at world 1"))
    argv = ["--sensor_noise", "1", "--seed", "7", "--num_envs", "1024", "--batch", "512"]
    with pytest.raises(_Stop):
        train.main(argv)
    args = train.parser().parse_args(argv)
    assert seeds == [7]
    cfg = made["env_cfg"]
    want = train.train_env_config(args)
    assert cfg.keys() == want.keys() and cfg["noise_seed"] == 7
    assert all(np.array_equal(np.asarray(cfg[k], dtype=object), np.asarray(want[k], dtype=object)) for k in cfg if k != "heightfield")
    assert (made["rank"], made["world"], made["device"], made["n"], made["agent"]) == (0, 1, 0, 1024, (49, 12, 0, 7))
    assert seen == dict(batch=512, gamma=train.GAMMA, tau=train.TAU, alpha=train.ALPHA, actor_lr=train.ACTOR_LR, critic_lr=train.CRITIC_LR,
                        world=1, seed_key=0)


def test_rank_seeds_and_noise_seed():
    from paddlerobotics_b200 import train
    a = train.parser().parse_args(["--sensor_noise", "1", "--seed", "7"])
    assert train.train_env_config(a)["noise_seed"] == 7 and train.train_env_config(a, 3)["noise_seed"] == 10


# every call in the rank's loop that places buffers or launches on a GPU: each must name the rank's device, or a rank r > 0 of an NCCL run
# (which sits on GPU r) would allocate on GPU 0
DEVICE_CALLS = ("VecQuadrupedalEnv", "PopulationEvaluator", "MujocoAgent", "ReplayMemory", "solutions_to_etg_device", "make_envs", "make_eval_env")


@pytest.mark.parametrize("module, function", [("train", "run"), ("pretrain", "pretrain")])
def test_the_rank_loop_names_its_device_on_every_device_call(module, function):
    import ast
    import importlib
    import inspect
    import textwrap
    src = textwrap.dedent(inspect.getsource(getattr(importlib.import_module("paddlerobotics_b200." + module), function)))
    calls = [c for c in ast.walk(ast.parse(src)) if isinstance(c, ast.Call) and isinstance(c.func, ast.Name) and c.func.id in DEVICE_CALLS]
    assert len(calls) >= 3
    for c in calls:
        kw = {k.arg: k.value for k in c.keywords}
        assert "device" in kw and isinstance(kw["device"], ast.Name) and kw["device"].id == "dev", (module, c.func.id, c.lineno)


def test_pretrain_resume_checks_the_saved_population(monkeypatch, tmp_path, capsys):
    """At W > 1 the divisibility check reads the saved run's --popsize, not this command line's default."""
    from paddlerobotics_b200 import dist_run, pretrain
    for k, v in (("RANK", "0"), ("WORLD_SIZE", "3"), ("LOCAL_RANK", "0")):
        monkeypatch.setenv(k, v)

    def group(*a, **k):
        raise _Stop
    monkeypatch.setattr(dist_run, "process_group", group)
    for pop, ok in ((48, True), (40, False)):
        path = str(tmp_path / ("state%d.pt" % pop))
        torch.save({"command": "pretrain", "args": vars(pretrain.parser().parse_args(["--popsize", str(pop), "--outdir", "o"]))}, path)
        if ok:
            with pytest.raises(_Stop):                   # past the argument checks: the process group is next
                pretrain.main(["--resume", path])
        else:
            with pytest.raises(SystemExit):
                pretrain.main(["--resume", path])
            assert "--popsize 40 must be divisible by the 3 ranks" in capsys.readouterr().err
