"""dynamic_train (the batched Dynamic_train.py) without a device: the restated ES solvers against the reference's own (tests/golden/
es_solvers.npz, written by make_es_solvers.py from ETGRL/alg/es.py through ES_ParallelModel.set_solver), the flag defaults, and the
inputs it refuses before any device work."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ALGS = ("ga", "ses", "pepg", "openes", "simples")


@pytest.fixture(scope="module")
def solvers():
    return np.load(os.path.join(GOLDEN, "es_solvers.npz"))


@pytest.mark.parametrize("alg", ALGS)
def test_solver_reproduces_the_reference_bit_for_bit(solvers, alg):
    """Same seed, same fitness: every asked population and every result() equal the reference's, for all rounds."""
    from paddlerobotics_b200.dynamic_train import make_solver
    g = solvers
    np.random.seed(int(g[alg + "_seed"]))
    s = make_solver(alg, int(g["popsize"]), float(g["sigma"]), num_params=int(g["num_params"]), sigma_decay=float(g["sigma_decay"]))
    rounds = g[alg + "_solutions"].shape[0]
    assert rounds >= 3
    for r in range(rounds):
        sol = s.ask()
        assert np.array_equal(sol, g[alg + "_solutions"][r]), (alg, r, np.abs(sol - g[alg + "_solutions"][r]).max())
        s.tell(g[alg + "_fitness"][r].copy())
        best, best_reward, curr_best_reward, sigma = s.result()
        assert np.array_equal(best, g[alg + "_best"][r]), (alg, r)
        assert best_reward == g[alg + "_best_reward"][r] and curr_best_reward == g[alg + "_curr_best_reward"][r], (alg, r)
        assert np.array_equal(np.asarray(sigma), g[alg + "_sigma"][r]), (alg, r)


def test_centered_ranks_are_float32():
    from paddlerobotics_b200.es import compute_centered_ranks
    y = compute_centered_ranks(np.array([3.0, -1.0, 2.0, 10.0, 0.5]))
    assert y.dtype == np.float32
    assert np.array_equal(y, np.array([0.25, -0.5, 0.0, 0.5, -0.25], dtype=np.float32))


def test_rank_fitness_forgets_the_best():
    """With rank_fitness, result()[0] is the best member of the CURRENT generation, even when an earlier one scored higher."""
    from paddlerobotics_b200.es import OpenES, PEPG
    for cls in (OpenES, PEPG):
        np.random.seed(0)
        s = cls(4, popsize=6, weight_decay=0.0)
        s.ask(); s.tell(np.array([0, 0, 0, 0, 0, 100.0]))
        sol = s.ask(); s.tell(np.array([1.0, 5.0, 2.0, 0.0, 3.0, 4.0]))
        assert np.array_equal(s.result()[0], sol[1]), cls.__name__


def test_vectorised_dynamics_rows_equal_the_per_vector_rows_bit_for_bit():
    """param2dynamic_rows over a population == dynamic_dict_to_row(param2dynamic_dict(p)) per vector, in range, beyond the [-1, 1] clip,
    at the clip and at zero."""
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict, param2dynamic_rows
    rng = np.random.default_rng(0)
    s = np.concatenate([rng.uniform(-1, 1, (300, 48)), rng.uniform(-3, 3, (100, 48)), rng.normal(0, 0.1, (100, 48)),
                        rng.choice([-1.0, 1.0, 0.0, -0.0, -0.98, 0.98, 1e-17, -1e-300, 0.5], (100, 48))])
    ref = np.array([dynamic_dict_to_row(param2dynamic_dict(x)) for x in s])
    rows = param2dynamic_rows(s)
    assert rows.shape == ref.shape and np.array_equal(rows.view(np.uint64), ref.view(np.uint64))


def test_flag_defaults_are_dynamic_train_s():
    """Dynamic_train.py:20-31, plus --data_dir and --seed."""
    from paddlerobotics_b200 import dynamic_train
    a = dynamic_train.parser().parse_args([])
    assert (a.outdir, a.suffix, a.steps, a.K, a.thread, a.sigma, a.alg, a.load, a.eval, a.gamma) == ("Dynamic", "exp0", 10000, 20, 2, 0.1, "ga", "", 0, 1)
    assert a.xparl == "172.18.188.13:8007"
    assert (a.data_dir, a.seed) == ("data/dynamic", 0)


def test_evaluator_config_is_make_env_ground_without_etg_keyword():
    from paddlerobotics_b200.dynamic_train import evaluator_config
    cfg = evaluator_config()
    assert "etg_enabled" not in cfg and cfg["heightfield"] is None
    assert cfg["joint_limits"] == 1 and cfg["knee_contacts"] == 1


def _write_data(d, rows=100, drop=None, short=None):
    from paddlerobotics_b200.dynamic_train import DATA_FILES, STATS
    os.makedirs(d, exist_ok=True)
    md = {}
    for key in ("exp", "ori", "height"):
        for s in STATS:
            n = rows - 1 if short == key + s else rows
            md[key + s] = np.ones((n, 12 if "motor" in s else 3))
        np.save(os.path.join(d, DATA_FILES[key]), np.zeros((rows - 1 if short == key else rows, 12)))
    np.savez(os.path.join(d, DATA_FILES["mean_dict"]), **md)
    if drop:
        os.remove(os.path.join(d, DATA_FILES[drop]))


def _refused(capsys, argv):
    from paddlerobotics_b200 import dynamic_train
    with pytest.raises(SystemExit) as e:
        dynamic_train.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


def test_load_data_accepts_the_four_files(tmp_path):
    from paddlerobotics_b200.dynamic_train import load_data
    _write_data(str(tmp_path))
    gait, md = load_data(str(tmp_path))
    assert set(gait) == {"exp", "ori", "height"} and len(md) == 12


def test_refuses_cma_naming_the_supported_algorithms(tmp_path, capsys):
    _write_data(str(tmp_path))
    err = _refused(capsys, ["--alg", "cma", "--data_dir", str(tmp_path)])
    assert "cma" in err and "ga, ses, pepg, openes, simples" in err


def test_refuses_eval_without_load(tmp_path, capsys):
    _write_data(str(tmp_path))
    err = _refused(capsys, ["--eval", "1", "--data_dir", str(tmp_path)])
    assert "--load" in err


@pytest.mark.parametrize("drop", ["mean_dict", "exp", "ori", "height"])
def test_refuses_a_missing_data_file_by_name(tmp_path, capsys, drop):
    from paddlerobotics_b200.dynamic_train import DATA_FILES
    _write_data(str(tmp_path), drop=drop)
    err = _refused(capsys, ["--data_dir", str(tmp_path)])
    assert DATA_FILES[drop] in err and "missing" in err


@pytest.mark.parametrize("short", ["exp", "height", "ori_motor_std", "height_drpy_mean"])
def test_refuses_a_table_or_statistic_shorter_than_100_rows(tmp_path, capsys, short):
    from paddlerobotics_b200.dynamic_train import DATA_FILES
    _write_data(str(tmp_path), short=short)
    err = _refused(capsys, ["--data_dir", str(tmp_path)])
    assert DATA_FILES[short if short in DATA_FILES else "mean_dict"] in err and "100" in err
