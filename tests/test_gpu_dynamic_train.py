"""dynamic_train (the batched Dynamic_train.py) on the GPU, on synthetic data: the real-robot statistics are not in the tree, so the gait
tables are slices of the shipped CPG table and the statistics are simulated under a planted parameter vector p*.  Also train.py's
--dynamic_param on the training and ES evaluator envs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
POSE = np.array([0, 0.9, -1.8] * 4)
T = 100
KEYS = ("exp", "ori", "height")
# a benign planted vector: leg-mass multipliers >= 0.75 (light legs can diverge at settle, DESIGN §6) and foot friction 0.8
P_STAR = np.random.default_rng(5).uniform(-0.25, 0.25, 48)
P_STAR[1] = 0.06


def gait_tables():
    tab = np.load(os.path.join(GOLDEN, "gait_action_list_CPG_stairstair7_12_3.npy")) + POSE
    return {k: tab[i * T:(i + 1) * T] for i, k in enumerate(KEYS)}


def planted_data(p_star, precision="f32"):
    """(gait, mean_dict): the means are p*'s own rollout of each table on the command's evaluator config; the stds are constants."""
    from paddlerobotics_b200.dynamic_train import evaluator_config
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    gait = gait_tables()
    env = VecQuadrupedalEnv(len(KEYS), precision=precision, etg_enabled=0, ring_depth=4, **evaluator_config())
    env.set_dynamics(np.repeat(dynamic_dict_to_row(param2dynamic_dict(p_star))[None], len(KEYS), 0))
    env.reset()
    motor, drpy = [], []
    for t in range(T):
        _, _, _, info = env.step(np.stack([gait[k][t] - POSE for k in KEYS]), donef=False)
        info = info.double().cpu().numpy()
        motor.append(info[:, 42:54]); drpy.append(info[:, 39:42])
    env.close()
    motor, drpy = np.array(motor), np.array(drpy)
    md = {}
    for i, k in enumerate(KEYS):
        md[k + "_motor_mean"], md[k + "_drpy_mean"] = motor[:, i], drpy[:, i]
        md[k + "_motor_std"], md[k + "_drpy_std"] = np.full((T, 12), 0.1), np.full((T, 3), 0.5)
    return gait, md


def write_data(d, gait, md):
    from paddlerobotics_b200.dynamic_train import DATA_FILES
    os.makedirs(d, exist_ok=True)
    np.savez(os.path.join(d, DATA_FILES["mean_dict"]), **md)
    for k in KEYS:
        np.save(os.path.join(d, DATA_FILES[k]), gait[k])
    return d


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    gait, md = planted_data(P_STAR)
    return write_data(str(tmp_path_factory.mktemp("dyn")), gait, md)


def _lines(out):
    return [json.loads(l) for l in out.splitlines() if l.startswith("{")]


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_planted_parameter_scores_exactly_30(precision):
    from paddlerobotics_b200.dynamic_train import evaluator_config
    from paddlerobotics_b200.es import DynamicsEvaluator
    gait, md = planted_data(P_STAR, precision)
    sols = np.stack([P_STAR, P_STAR + 0.2, np.zeros(48), -P_STAR])
    ev = DynamicsEvaluator(4, gait, md, keys=("exp", "ori"), precision=precision, **evaluator_config())
    rew = ev.evaluate(sols).double().cpu().numpy()
    assert rew[0] == 30.0 and (rew[1:] < 30.0).all(), rew
    h = DynamicsEvaluator(1, gait, md, keys=("height",), precision=precision, **evaluator_config())
    assert float(h.evaluate(P_STAR[None])[0]) == 30.0
    ev.env.close(); h.env.close()


def test_ga_end_to_end(tmp_path, capsys, data_dir):
    """Ten epochs of --alg ga: the files, the lines, the rewards of DynamicsEvaluator on the same solutions bit for bit, and progress."""
    from paddlerobotics_b200 import dynamic_train
    from paddlerobotics_b200.dynamic_train import DATA_FILES, evaluator_config, load_data, make_solver
    from paddlerobotics_b200.es import DynamicsEvaluator
    out = str(tmp_path / "out")
    dynamic_train.main(["--alg", "ga", "--steps", "10", "--data_dir", data_dir, "--outdir", out, "--suffix", "s"])
    lines = _lines(capsys.readouterr().out)
    epochs = [r for r in lines if "reward_max" in r]
    evals = [r for r in lines if "eval_reward" in r]
    assert [r["epoch"] for r in epochs] == list(range(10)) and [r["epoch"] for r in evals] == [5]
    params = [np.load(os.path.join(out, "s", "dynamic_param%d.npy" % e)) for e in range(10)]
    assert all(p.shape == (48,) and p.dtype == np.float64 for p in params)
    assert sorted(os.listdir(os.path.join(out, "s"))) == sorted("dynamic_param%d.npy" % e for e in range(10))
    # the same epochs by hand
    gait, md = load_data(data_dir)
    np.random.seed(0)
    solver = make_solver("ga", 40, 0.1)
    ev = DynamicsEvaluator(40, gait, md, keys=("exp", "ori"), **evaluator_config())
    for e in range(10):
        rew = ev.evaluate(solver.ask()).double().cpu().numpy()
        solver.tell(rew)
        r = epochs[e]
        assert (r["reward_max"], r["reward_mean"], r["reward_min"], r["reward_std"]) == (rew.max(), rew.mean(), rew.min(), rew.std()), e
        assert np.array_equal(solver.result()[0], params[e]) and r["sigma"] == solver.result()[3]
    ev.env.close()
    assert epochs[-1]["best_reward"] > epochs[0]["best_reward"], (epochs[0], epochs[-1])
    # --eval 1 --load of epoch 5's vector gives the line of epoch 5's height evaluation
    rec = dynamic_train.main(["--eval", "1", "--load", os.path.join(out, "s", "dynamic_param5.npy"), "--data_dir", data_dir])
    assert rec[0]["eval_reward"] == evals[0]["eval_reward"]
    assert _lines(capsys.readouterr().out) == rec
    assert DATA_FILES["mean_dict"] in os.listdir(data_dir)


@pytest.mark.parametrize("alg", ["ga", "ses", "pepg", "openes", "simples"])
def test_every_alg_runs_two_epochs(tmp_path, capsys, data_dir, alg):
    from paddlerobotics_b200 import dynamic_train
    log = dynamic_train.main(["--alg", alg, "--steps", "2", "--data_dir", data_dir, "--outdir", str(tmp_path)])
    assert [r["epoch"] for r in log] == [0, 1] and all(np.isfinite(r["reward_max"]) and np.isfinite(r["sigma"]) for r in log), log
    assert _lines(capsys.readouterr().out) == log
    assert np.load(str(tmp_path / "exp0" / "dynamic_param1.npy")).shape == (48,)


def test_height_reward_matches_the_float64_oracle(data_dir):
    """One vector on the `height` table: f64 engine == oracle rollout on the same config + the NumPy restatement of loss_func, to 1e-6."""
    from oracle import oracle as O
    from paddlerobotics_b200.dynamic_train import evaluator_config, load_data
    from paddlerobotics_b200.es import DynamicsEvaluator
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    gait, md = load_data(data_dir)
    p = P_STAR + np.random.default_rng(9).uniform(-0.05, 0.05, 48)
    cfg = evaluator_config()
    ev = DynamicsEvaluator(1, gait, md, keys=("height",), precision="f64", **cfg)
    rew = float(ev.evaluate(p[None])[0])
    ev.env.close()
    okeys = {f[0] for f in O.Config._fields_}
    o = O.OracleEnv(O.default_config(etg_enabled=0, **{k: v for k, v in cfg.items() if k in okeys}), dynamic_dict_to_row(param2dynamic_dict(p)))
    o.reset()
    motor, drpy = [], []
    for t in range(T):
        _, _, _, info = o.step(gait["height"][t] - POSE)
        motor.append(info[42:54]); drpy.append(info[39:42])
    motor, drpy = np.array(motor), np.array(drpy)
    lm = np.max(np.mean((motor - md["height_motor_mean"][:T]) ** 2 / md["height_motor_std"][:T] ** 2, axis=0))     # Dynamic_parallel_model.py:29-41
    ld = np.max(np.mean((drpy - md["height_drpy_mean"][:T]) ** 2 / md["height_drpy_std"][:T] ** 2, axis=0))
    ref = 30 - (ld + lm) / 2.0
    assert ref < 30.0 and abs(rew - ref) < 1e-6, (rew, ref)


def test_train_dynamic_param_reaches_training_and_es_envs(tmp_path, etg_default):
    """train.py --dynamic_param: after reset, the training env and the ES evaluator's env observe what a VecQuadrupedalEnv with
    set_dynamics(row) observes, bit for bit, and not what the nominal dynamics give."""
    import torch
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    w, b = etg_default
    p = np.random.default_rng(3).uniform(-0.25, 0.25, 48)
    path = str(tmp_path / "dynamic_param7.npy")
    np.save(path, p)
    args = train.parser().parse_args(["--dynamic_param", path, "--num_envs", "8", "--popsize", "4", "--es_rollouts", "2"])
    env_cfg = train.env_config(args)
    env, ev = train.make_envs(args, env_cfg)
    ref = VecQuadrupedalEnv(8, **env_cfg)
    ref.set_dynamics(np.repeat(dynamic_dict_to_row(param2dynamic_dict(p))[None], 8, 0))
    nominal = VecQuadrupedalEnv(8, **env_cfg)
    o_ref, o_nom = ref.reset(w, b).clone(), nominal.reset(w, b).clone()
    assert torch.equal(env.reset(w, b), o_ref)
    assert torch.equal(ev.env.reset(w, b), o_ref)
    assert not torch.equal(o_ref, o_nom)
    # and the default path stays nominal
    env0, ev0 = train.make_envs(train.parser().parse_args(["--num_envs", "8", "--popsize", "4", "--es_rollouts", "2"]), env_cfg)
    assert torch.equal(env0.reset(w, b), o_nom) and torch.equal(ev0.env.reset(w, b), o_nom)
    for e in (env, ev.env, ref, nominal, env0, ev0.env):
        e.close()


def test_sharded_rewards_equal_single_gpu(tmp_path, capsys, data_dir):
    """Under torchrun on two GPUs, the command's epoch lines (rewards of the all-gathered shards) equal a single-GPU run's bit for bit."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from paddlerobotics_b200 import dynamic_train
    argv = ["--alg", "pepg", "--steps", "2", "--data_dir", data_dir]
    single = dynamic_train.main(argv + ["--outdir", str(tmp_path / "one")])
    capsys.readouterr()
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                          "--master-port", "29547", "-m", "paddlerobotics_b200.dynamic_train"] + argv + ["--outdir", str(tmp_path / "two")],
                         capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert _lines(out.stdout) == single
