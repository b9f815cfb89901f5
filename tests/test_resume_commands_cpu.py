"""--save_state / --resume of pretrain, dynamic_train and bctrain without a device: the shared writer and argument merge (run_state, and the
same functions through train), every refusal of a resume, and the state round trip of all five ES solvers."""
import os

import numpy as np
import pytest
import torch

from paddlerobotics_b200 import bctrain, dynamic_train, pretrain, run_state, train

COMMANDS = {"pretrain": pretrain, "dynamic_train": dynamic_train, "bctrain": bctrain}
FREE = {"pretrain": ["--max_steps", "5", "--outdir", "o2", "--suffix", "z", "--save_state", "0"],
        "dynamic_train": ["--steps", "5", "--outdir", "o2", "--suffix", "z", "--save_state", "0"],
        "bctrain": ["--max_steps", "5", "--outdir", "o2", "--suffix", "z", "--save_state", "0"]}
CHANGED = {"pretrain": (["--popsize", "20", "--seed", "3"], "--popsize, --seed"), "dynamic_train": (["--alg", "pepg"], "--alg"),
           "bctrain": (["--num_envs", "64", "--memory", "5000"], "--memory, --num_envs")}
CONFLICTS = {"pretrain": [(["--load", "x.npz"], "--load"), (["--ETG_path", "g.npz"], "--ETG_path"), (["--eval", "1"], "--eval 1")],
             "dynamic_train": [(["--load", "x.npy"], "--load"), (["--eval", "1"], "--eval 1")],
             "bctrain": [(["--load", "x.pt"], "--load"), (["--ETG_path", "g.npz"], "--ETG_path"), (["--eval", "1"], "--eval 1")]}


def _saved(tmp_path, command, **over):
    """A state.pt of `command` whose only fields a resume reads before device work are `command` and `args` (train: `args` only)."""
    mod = train if command == "train" else COMMANDS[command]
    args = vars(mod.parser().parse_args(["--outdir", str(tmp_path), "--save_state", "1"]))
    args.update(over)
    path = str(tmp_path / ("%s_state.pt" % command))
    torch.save({"args": args} if command == "train" else {"command": command, "args": args}, path)
    return path


@pytest.fixture
def no_device(monkeypatch):
    """Any device work fails the test: the refusals must come first."""
    fail = lambda *a, **k: pytest.fail("device work before an argument error")
    monkeypatch.setattr(pretrain, "pretrain", fail)
    monkeypatch.setattr(pretrain, "evaluate", fail)
    monkeypatch.setattr(dynamic_train, "run", fail)
    monkeypatch.setattr(dynamic_train, "load_data", fail)
    monkeypatch.setattr(bctrain, "MujocoAgent", fail)
    monkeypatch.setattr(bctrain, "etg_of_path", fail)
    monkeypatch.setattr(train, "VecQuadrupedalEnv", fail)
    monkeypatch.setattr(train, "make_envs", fail)


@pytest.mark.parametrize("command", sorted(COMMANDS))
def test_flag_defaults(command):
    args = COMMANDS[command].parser().parse_args([])
    assert args.save_state == 0 and args.resume == ""


@pytest.mark.parametrize("command", sorted(COMMANDS))
def test_save_state_needs_outdir(no_device, capsys, command):
    with pytest.raises(SystemExit):
        COMMANDS[command].main(["--save_state", "1", "--outdir", ""])
    assert "needs --outdir" in capsys.readouterr().err


@pytest.mark.parametrize("command", sorted(COMMANDS))
def test_resume_refuses_changed_arguments_naming_them(no_device, tmp_path, capsys, command):
    path = _saved(tmp_path, command)
    extra, named = CHANGED[command]
    with pytest.raises(SystemExit):
        COMMANDS[command].main(["--resume", path] + extra)
    err = capsys.readouterr().err
    assert "differ from the saved run" in err and named in err


@pytest.mark.parametrize("command,extra,named", [(c, e, n) for c in sorted(COMMANDS) for e, n in CONFLICTS[c]])
def test_resume_conflicts_are_argument_errors(no_device, tmp_path, capsys, command, extra, named):
    path = _saved(tmp_path, command)
    with pytest.raises(SystemExit):
        COMMANDS[command].main(["--resume", path] + extra)
    err = capsys.readouterr().err
    assert "cannot be combined with" in err and named in err


ALL = ("train", "pretrain", "dynamic_train", "bctrain")


@pytest.mark.parametrize("writer,reader", [(w, r) for w in ALL for r in ALL if w != r])
def test_a_state_file_of_another_command_is_refused(no_device, tmp_path, capsys, writer, reader):
    path = _saved(tmp_path, writer)
    mod = train if reader == "train" else COMMANDS[reader]
    with pytest.raises(SystemExit):
        mod.main(["--resume", path])
    assert "a state file of %s, not of %s" % (writer, reader) in capsys.readouterr().err


@pytest.mark.parametrize("command", sorted(COMMANDS))
def test_resume_takes_saved_arguments_and_the_free_flags(tmp_path, command):
    mod = COMMANDS[command]
    path = _saved(tmp_path, command, seed=7)
    saved = torch.load(path, weights_only=False)
    assert run_state.load_state(mod.parser(), path, command) is not None
    argv = ["--resume", path, "--seed", "7"] + FREE[command]                 # an equal value may be repeated
    args = run_state.resume_args(mod.parser(), mod.parser, argv, saved["args"], mod.RESUME_FREE, (), "the run")
    budget = "steps" if command == "dynamic_train" else "max_steps"
    assert args.seed == 7 and getattr(args, budget) == 5 and (args.outdir, args.suffix, args.save_state, args.resume) == ("o2", "z", 0, path)
    for k, v in saved["args"].items():
        if k not in mod.RESUME_FREE:
            assert getattr(args, k) == v, k


def test_train_keeps_its_resume_surface(tmp_path):
    """train.write_atomic, train.resume_args and train.RESUME_FREE are the shared module's writer and merge, with train's flags."""
    assert train.write_atomic is run_state.write_atomic
    assert train.RESUME_FREE == ("max_steps", "log_every", "outdir", "suffix", "save_state", "resume")
    path = _saved(tmp_path, "train", seed=7)
    saved = torch.load(path, weights_only=False)
    assert run_state.command_of(saved) == "train" and run_state.load_state(train.parser(), path, "train")["args"] == saved["args"]
    args = train.resume_args(train.parser(), ["--resume", path, "--log_every", "3"], saved["args"])
    assert args.seed == 7 and args.log_every == 3
    with pytest.raises(SystemExit):
        train.resume_args(train.parser(), ["--resume", path, "--log_every", "3", "--batch", "1"], saved["args"])


def test_shared_writer_keeps_the_previous_file_when_interrupted(tmp_path, monkeypatch):
    path = str(tmp_path / "state.pt")
    run_state.write_atomic(path, {"it": 1})

    class Boom:
        def __reduce__(self):
            raise RuntimeError("interrupted mid-write")
    with pytest.raises(RuntimeError):
        run_state.write_atomic(path, {"it": 2, "boom": Boom()})
    assert torch.load(path)["it"] == 1
    run_state.write_atomic(path, {"it": 3})
    assert torch.load(path)["it"] == 3 and not os.path.exists(path + ".tmp")


def _solver(alg):
    if alg == "pretrain":
        from paddlerobotics_b200.es import SimpleGA
        return SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=10, param=np.zeros(12))
    return dynamic_train.make_solver(alg, 20, 0.1)


def _fitness(sol, k):
    return -np.square(sol - 0.05 * k).sum(1)


@pytest.mark.parametrize("alg", list(dynamic_train.ALGS) + ["pretrain"])
def test_solver_round_trip_asks_the_same_populations(tmp_path, alg):
    """After a load the next ask() equals the saved solver's bit for bit, and so do the tell() and ask() after it (the Adam optimiser of
    openes / pepg moves the loaded solver's mu, not a copy's)."""
    np.random.seed(5)
    s = _solver(alg)
    for k in range(4):
        s.tell(_fitness(s.ask(), k))
    torch.save(s.state_dict(), tmp_path / "solver.pt")
    sd = torch.load(tmp_path / "solver.pt", weights_only=False)         # through a file, as --resume reads it
    cont = []
    for k in range(4, 7):
        sol = s.ask()
        cont.append(sol)
        s.tell(_fitness(sol, k))
    np.random.seed(123)                                                  # another process: a fresh solver, another RNG state
    s2 = _solver(alg)
    s2.load_state_dict(sd)
    for k, want in zip(range(4, 7), cont):
        sol = s2.ask()
        np.testing.assert_array_equal(sol, want)
        s2.tell(_fitness(sol, k))
    for a, b in zip(s.result(), s2.result()):
        np.testing.assert_array_equal(a, b)
    if hasattr(s2, "optimizer"):
        assert s2.optimizer.pi is s2 and s2.optimizer.t == s.optimizer.t

