"""--save_state / --resume of train.py without a device: the flag defaults, the argument errors of a resume, the SimpleGA + NumPy RNG
round trip, and the atomic state writer."""
import os

import numpy as np
import pytest
import torch


def _no_device(monkeypatch):
    from paddlerobotics_b200 import train
    fail = lambda *a, **k: pytest.fail("an env was constructed")
    monkeypatch.setattr(train, "VecQuadrupedalEnv", fail)
    monkeypatch.setattr(train, "make_envs", fail)


def _saved_state(tmp_path, **over):
    """A state.pt whose only field a resume reads before device work is `args`."""
    from paddlerobotics_b200 import train
    args = vars(train.parser().parse_args(["--num_envs", "64", "--batch", "128", "--outdir", str(tmp_path), "--save_state", "1"]))
    args.update(over)
    path = str(tmp_path / "state.pt")
    torch.save({"args": args}, path)
    return path


def test_flag_defaults():
    from paddlerobotics_b200 import train
    args = train.parser().parse_args([])
    assert args.save_state == 0 and args.resume == ""


def test_save_state_needs_outdir(monkeypatch):
    from paddlerobotics_b200 import train
    _no_device(monkeypatch)
    with pytest.raises(SystemExit):
        train.main(["--save_state", "1"])


@pytest.mark.parametrize("extra,named", [(["--batch", "256"], "--batch"), (["--seed", "3", "--memory", "5000"], "--memory, --seed"),
                                         (["--graph_iter", "0"], "--graph_iter")])
def test_resume_refuses_changed_arguments_naming_them(monkeypatch, tmp_path, capsys, extra, named):
    from paddlerobotics_b200 import train
    _no_device(monkeypatch)
    path = _saved_state(tmp_path)
    with pytest.raises(SystemExit):
        train.main(["--resume", path] + extra)
    err = capsys.readouterr().err
    assert "differ from the saved run" in err and named in err


@pytest.mark.parametrize("extra,named", [(["--load", "x.pt"], "--load"), (["--ETG_path", "g.npz"], "--ETG_path"), (["--eval", "1"], "--eval 1")])
def test_resume_conflicts_are_argument_errors(monkeypatch, tmp_path, capsys, extra, named):
    from paddlerobotics_b200 import train
    _no_device(monkeypatch)
    path = _saved_state(tmp_path)
    with pytest.raises(SystemExit):
        train.main(["--resume", path] + extra)
    assert named in capsys.readouterr().err


def test_resume_takes_saved_arguments_and_the_free_flags(tmp_path):
    from paddlerobotics_b200 import train
    path = _saved_state(tmp_path, seed=7, memory=5000)
    p = train.parser()
    argv = ["--resume", path, "--max_steps", "999", "--log_every", "3", "--suffix", "b", "--outdir", "o2", "--save_state", "0", "--batch", "128"]
    args = train.resume_args(p, argv, torch.load(path, weights_only=False)["args"])
    assert (args.seed, args.memory, args.num_envs, args.batch) == (7, 5000, 64, 128)        # saved; an equal value may be repeated
    assert (args.max_steps, args.log_every, args.suffix, args.outdir, args.save_state, args.resume) == (999, 3, "b", "o2", 0, path)


def test_simple_ga_and_numpy_rng_round_trip():
    from paddlerobotics_b200.es import SimpleGA
    np.random.seed(5)
    ga = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=10, param=np.zeros(12))
    for _ in range(3):                                   # decayed sigma, a non-trivial elite set and best parameters
        sol = ga.ask()
        ga.tell(-np.square(sol).sum(1))
    sd = ga.state_dict()
    nxt = ga.ask()
    np.random.seed(123)                                  # another process: fresh solver, other RNG state
    ga2 = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=10, param=np.zeros(12))
    ga2.load_state_dict(sd)
    assert ga2.sigma == sd["attrs"]["sigma"] and ga2.sigma < 0.02
    np.testing.assert_array_equal(ga2.elite_params, sd["attrs"]["elite_params"])
    np.testing.assert_array_equal(ga2.ask(), nxt)


def test_atomic_writer_keeps_the_previous_file_when_interrupted(tmp_path, monkeypatch):
    from paddlerobotics_b200 import train
    path = str(tmp_path / "state.pt")
    train.write_atomic(path, {"it": 1, "x": torch.arange(4)})
    assert not os.path.exists(path + ".tmp")

    class Boom:
        def __reduce__(self):
            raise RuntimeError("interrupted mid-write")
    with pytest.raises(RuntimeError):
        train.write_atomic(path, {"it": 2, "big": torch.zeros(1 << 16), "boom": Boom()})
    assert torch.load(path)["it"] == 1

    def no_rename(*a):
        raise KeyboardInterrupt
    monkeypatch.setattr(os, "replace", no_rename)         # written and fsynced, stopped before the rename
    with pytest.raises(KeyboardInterrupt):
        train.write_atomic(path, {"it": 3})
    assert torch.load(path)["it"] == 1
    monkeypatch.undo()
    train.write_atomic(path, {"it": 4})
    assert torch.load(path)["it"] == 4
