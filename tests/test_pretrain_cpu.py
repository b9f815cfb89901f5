"""pretrain (the batched ETGRL/pretrain.py), train.py's --ETG_path rule and env_test without a device: the flag defaults against
pretrain.py:292-330, the options refused before any device work, argument errors, the evaluation / checkpoint cadence, and initial_etg."""
import argparse

import numpy as np
import pytest

# pretrain.py:292-329 (flag defaults; popsize is type=float there and an int here) and :34-37 (module constants that became flags)
REFERENCE_DEFAULTS = {
    "outdir": "train_log", "max_steps": 1e7, "epsilon": 0.4, "gamma": 0.95, "sigma": 0.02, "sigma_decay": 0.99, "popsize": 40,
    "random_dynamic": 0, "random_force": 0, "task_mode": "stairstair", "step_y": 0.05, "load": "", "eval": 0, "render": 0, "suffix": "exp0",
    "random": 0, "normal": 1, "vel_d": 0.5, "ETG_T": 0.5, "reward_p": 5, "footheight": 0.1, "steplen": 0.05, "ETG": 1, "ETG_T2": 0.5,
    "e_step": 400, "act_mode": "traj", "ETG_path": "None", "ETG_H": 20, "stand": 0, "torso": 1.5, "up": 0.6, "tau": 0.07, "feet": 0.3,
    "badfoot": 0.1, "footcontact": 0.1, "enable_action_filter": 0, "x_noise": 0,
    # ES_TRAIN_STEPS, EVAL_EVERY_STEPS, and the one episode per solution of pretrain.py:228-232
    "es_train_steps": 10, "eval_every_steps": 1e4, "es_rollouts": 1,
}


def test_flag_defaults_are_the_reference_values():
    from paddlerobotics_b200 import pretrain
    a = pretrain.parser().parse_args([])
    for k, v in REFERENCE_DEFAULTS.items():
        assert getattr(a, k) == v, (k, getattr(a, k), v)
    assert isinstance(a.popsize, int) and isinstance(pretrain.parser().parse_args(["--popsize", "8"]).popsize, int)
    assert a.dynamic_param == "" and a.eval_envs == 1


def _no_device(monkeypatch, module):
    import torch

    def no_device(*a, **k):
        raise AssertionError("device touched before the option check")
    monkeypatch.setattr(torch.cuda, "_lazy_init", no_device)
    monkeypatch.setattr(module, "pretrain", no_device)
    monkeypatch.setattr(module, "evaluate", no_device)


@pytest.mark.parametrize("flags", [["--random_dynamic", "1"], ["--random_force", "1"], ["--x_noise", "1"], ["--render", "1"], ["--stand", "0.5"],
                                   ["--ETG_H", "16"], ["--ETG", "0"], ["--ETG_T2", "0.4"], ["--act_mode", "pose"], ["--act_mode", "torque"]])
def test_unsupported_flags_raise_before_any_device_work(flags, monkeypatch):
    from paddlerobotics_b200 import pretrain
    _no_device(monkeypatch, pretrain)
    with pytest.raises(NotImplementedError):
        pretrain.main(flags)
    with pytest.raises(NotImplementedError):
        pretrain.main(flags + ["--eval", "1", "--load", "x.npz"])


def test_ignored_flags_are_accepted(monkeypatch):
    from paddlerobotics_b200 import pretrain
    seen = []
    monkeypatch.setattr(pretrain, "pretrain", lambda args: seen.append(args))
    pretrain.main(["--epsilon", "0.1", "--gamma", "0.5", "--random", "1", "--e_step", "100"])
    assert len(seen) == 1 and seen[0].random == 1


def test_argument_errors(monkeypatch, tmp_path):
    from paddlerobotics_b200 import pretrain, train
    _no_device(monkeypatch, pretrain)
    with pytest.raises(SystemExit):
        pretrain.main(["--eval", "1"])
    with pytest.raises(SystemExit):
        pretrain.main(["--popsize", "0"])
    with pytest.raises(SystemExit):                 # int(0.1 * 9) = 0 elites: SimpleGA.ask has no parent to draw
        pretrain.main(["--popsize", "9"])
    monkeypatch.setattr(train, "evaluate", lambda *a: pytest.fail("reached the evaluation"))
    monkeypatch.setattr(train, "make_envs", lambda *a, **k: pytest.fail("reached the training set-up"))
    npz = str(tmp_path / "g.npz")
    np.savez(npz, w=np.zeros((3, 20)), b=np.zeros(3), param=np.zeros(12))
    for extra in ([], ["--eval", "1"]):
        with pytest.raises(SystemExit):
            train.main(["--ETG_path", npz, "--load", str(tmp_path / "itr_0.pt")] + extra)
        with pytest.raises(SystemExit):     # the rule is about the flags, not about whether the file exists
            train.main(["--ETG_path", str(tmp_path / "missing.npz"), "--load", str(tmp_path / "itr_0.pt")] + extra)


def test_env_test_refuses_a_missing_gait(tmp_path):
    from paddlerobotics_b200 import env_test
    with pytest.raises(SystemExit):
        env_test.main(["--load", str(tmp_path / "missing.npz")])
    a = env_test.parser().parse_args([])
    assert (a.load, a.video, a.task, a.suffix, a.save, a.step_y) == ("data/origin_ETG/ESStair_origin.npz", 0, "stairstair", "exp", 0, 0.05)


def reference_cadence(round_totals, every):
    """pretrain.py:258-277 as written, counted per round: the while loop evaluates once per multiple, then one np.savez per round that
    entered the if.  Returns [(round, file name, evaluations the reference runs)]."""
    out, test_flag = [], 0
    for r, total in enumerate(round_totals):
        if (total + 1) // every >= test_flag:
            evals = 0
            while (total + 1) // every >= test_flag:
                test_flag += 1
                evals += 1
            out.append((r, "itr_{:d}.npz".format(int(total)), evals))
    return out


@pytest.mark.parametrize("every", [10000, 4000, 1])
def test_round_and_checkpoint_cadence(every):
    from paddlerobotics_b200 import pretrain
    rng = np.random.default_rng(every)
    totals = list(np.cumsum(rng.integers(1, 16040, 40)))            # a round: 10 generations of 40 x 1..401 steps
    ref = reference_cadence(totals, every)
    ours = pretrain.checkpoint_names(totals, every)
    assert ours == [(r, name) for r, name, _ in ref]                   # the same rounds write the same files ...
    assert ref[0][0] == 0                                              # ... the first round always evaluates ...
    if every == 1:
        assert any(e > 1 for _, _, e in ref)                           # ... and one evaluation stands for the reference's repeated ones


def test_cadence_at_the_multiples():
    from paddlerobotics_b200 import pretrain
    assert pretrain.checkpoint_names([5000, 9998, 9999, 25000, 26000, 45000], 10000) == [
        (0, "itr_5000.npz"), (2, "itr_9999.npz"), (3, "itr_25000.npz"), (5, "itr_45000.npz")]
    assert pretrain.eval_due(0, 0, 10000) == (True, 1)
    assert pretrain.eval_due(9998, 1, 10000) == (False, 1)


def _args(path, ETG_T=0.5, footheight=0.1, steplen=0.05):
    return argparse.Namespace(ETG_path=path, ETG_T=ETG_T, footheight=footheight, steplen=steplen)


def _prior():
    from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w0, b0, prior = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    return layer, w0, b0, prior


@pytest.mark.parametrize("path", ["None", "", None, "does/not/exist.npz"])
def test_initial_etg_without_a_file_is_todays_start(path, tmp_path):
    from paddlerobotics_b200.train import initial_etg
    _, w0, b0, _ = _prior()
    before = set(tmp_path.iterdir())
    param, w, b = initial_etg(_args(path if path != "does/not/exist.npz" else str(tmp_path / path.replace("/", "_"))))
    assert np.array_equal(param, np.zeros(12)) and np.array_equal(w, w0) and np.array_equal(b, b0)
    assert set(tmp_path.iterdir()) == before                           # no data/zero_param.npz is written


@pytest.mark.parametrize("shape", [(12,), (6, 2), (1, 12)])
def test_initial_etg_from_a_file(shape, tmp_path):
    from paddlerobotics_b200.etg import Opt_with_points
    from paddlerobotics_b200.train import initial_etg
    layer, w0, b0, prior = _prior()
    p = np.random.default_rng(1).uniform(-0.02, 0.02, 12)
    path = str(tmp_path / "g.npz")
    np.savez(path, w=np.ones((3, 20)), b=np.ones(3), param=p.reshape(shape))
    param, w, b = initial_etg(_args(path))
    assert param.shape == (12,) and np.array_equal(param, p)
    rw, rb, _ = Opt_with_points(ETG=layer, ETG_T=0.5, w0=w0, b0=b0, points=prior + p.reshape(-1, 2))
    assert np.abs(w - rw).max() <= 1e-12 and np.abs(b - rb).max() <= 1e-12
    assert np.abs(w - w0).max() > 1e-6                                  # the file moved the gait


@pytest.mark.parametrize("bad", [np.zeros(10), np.zeros((6, 3)), np.zeros(48)])
def test_initial_etg_rejects_other_sizes(bad, tmp_path):
    from paddlerobotics_b200.train import initial_etg
    path = str(tmp_path / "bad.npz")
    np.savez(path, param=bad)
    with pytest.raises(ValueError, match="bad.npz"):
        initial_etg(_args(path))
    np.savez(str(tmp_path / "nop.npz"), w=np.zeros((3, 20)))
    with pytest.raises(ValueError, match="nop.npz"):
        initial_etg(_args(str(tmp_path / "nop.npz")))
