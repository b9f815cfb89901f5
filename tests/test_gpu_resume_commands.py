"""--save_state / --resume of pretrain, dynamic_train and bctrain on the GPU: a run stopped after K rounds (epochs, iterations) and resumed to
2K against the run that was never stopped.  Each test first shows that two uninterrupted runs agree bit for bit over their common part
(the stopped run is one of them), which is what a bit-for-bit resume rests on."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_dynamic_train import P_STAR, planted_data, write_data
from test_gpu_resume import _same, _step

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(path):
    import torch
    return torch.load(path, weights_only=False)


def _same_states(a, b):
    """The state files of two runs agree bit for bit except for the arguments (outdir, budget)."""
    sa, sb = _load(os.path.join(a, "state.pt")), _load(os.path.join(b, "state.pt"))
    assert sa["command"] == sb["command"]
    sa.pop("args"); sb.pop("args")
    _same(sa, sb)
    return sa


def _same_npy_files(a, b, prefix, suffix):
    fa = sorted(f for f in os.listdir(a) if f.startswith(prefix) and f.endswith(suffix))
    assert fa and fa == sorted(f for f in os.listdir(b) if f.startswith(prefix) and f.endswith(suffix))
    for f in fa:
        if suffix == ".npy":
            x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), f
        else:
            with np.load(os.path.join(a, f)) as za, np.load(os.path.join(b, f)) as zb:
                assert sorted(za.files) == sorted(zb.files)
                for k in za.files:
                    assert za[k].tobytes() == zb[k].tobytes(), (f, k)
    return fa


# ---- pretrain: every round evaluates (--eval_every_steps 1), writes itr_*.npz and saves the state
PRE = ["--popsize", "10", "--es_train_steps", "2", "--task_mode", "ground", "--eval_every_steps", "1", "--suffix", "s", "--save_state", "1",
       "--seed", "3", "--sigma", "0.05"]


def test_pretrain_resume_equals_the_uninterrupted_run(tmp_path):
    import torch
    from paddlerobotics_b200 import pretrain
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    full = pretrain.main(PRE + ["--max_steps", "24000", "--outdir", a])
    ends = [r["env_steps"] for r in full if "checkpoint" in r]           # env steps at the end of each round
    assert len(ends) >= 4, ends
    k = len(ends) // 2
    part = pretrain.main(PRE + ["--max_steps", str(ends[k - 1]), "--outdir", b])
    assert part == full[:len(part)] and sum("checkpoint" in r for r in part) == k          # two uninterrupted runs agree
    saved = _load(os.path.join(b, "s", "state.pt"))
    assert saved["command"] == "pretrain" and saved["loop"]["env_steps"] == ends[k - 1] and saved["loop"]["es_step"] == 2 * k
    torch.manual_seed(12345); np.random.seed(12345)                                        # the state must bring NumPy's RNG back
    rest = pretrain.main(["--resume", os.path.join(b, "s", "state.pt"), "--max_steps", "24000", "--outdir", b])
    assert rest == full[len(part):]
    _same_npy_files(os.path.join(a, "s"), os.path.join(b, "s"), "itr_", ".npz")
    sa = _same_states(os.path.join(a, "s"), os.path.join(b, "s"))
    assert not sa["solver"]["attrs"]["first_iteration"]


# ---- dynamic_train: saves after epochs 5 and 10 (height evaluations) and after the last epoch
@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    gait, md = planted_data(P_STAR)
    return write_data(str(tmp_path_factory.mktemp("dyn")), gait, md)


@pytest.mark.parametrize("alg", ["ga", "ses", "pepg", "openes", "simples"])
def test_dynamic_train_resume_equals_the_uninterrupted_run(tmp_path, capsys, data_dir, alg):
    import torch
    from paddlerobotics_b200 import dynamic_train
    base = ["--alg", alg, "--K", "5", "--thread", "2", "--data_dir", data_dir, "--suffix", "s", "--save_state", "1", "--seed", "9"]
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    full = dynamic_train.main(base + ["--steps", "12", "--outdir", a])
    part = dynamic_train.main(base + ["--steps", "6", "--outdir", b])
    assert part == full[:len(part)] and part[-1]["epoch"] == 5                              # two uninterrupted runs agree
    saved = _load(os.path.join(b, "s", "state.pt"))
    assert saved["command"] == "dynamic_train" and saved["epoch"] == 6
    torch.manual_seed(12345); np.random.seed(12345)
    rest = dynamic_train.main(["--resume", os.path.join(b, "s", "state.pt"), "--steps", "12", "--outdir", b])
    assert rest == full[len(part):] and rest[0]["epoch"] == 6
    files = _same_npy_files(os.path.join(a, "s"), os.path.join(b, "s"), "dynamic_param", ".npy")
    assert len(files) == 12
    assert _same_states(os.path.join(a, "s"), os.path.join(b, "s"))["epoch"] == 12
    capsys.readouterr()


# ---- bctrain
N = 64
WALL = ("env_steps_per_s",)


def _expert_files(tmp_path):
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.train import etg_prior
    _, w, b, _ = etg_prior()
    MujocoAgent(49, 12, seed=1).save(str(tmp_path / "expert.pt"))
    np.savez(tmp_path / "expert.npz", w=w, b=b)
    return str(tmp_path / "expert.pt"), str(tmp_path / "expert.npz")


def _bc_base(tmp_path, warm):
    pt, npz = _expert_files(tmp_path)
    base = ["--ref_agent", pt, "--ETG_path", npz, "--num_envs", str(N), "--memory", "20000", "--eval_every_steps", str(10 * N), "--eval_envs", "2",
            "--suffix", "s", "--save_state", "1", "--seed", "4"]
    if warm:                                                 # the ring never reaches --warmup: random actions, no BC update
        return base + ["--warmup", "1000000"]
    return base + ["--batch", "128", "--train_per_time", "2", "--graph_steps", "4"]


def _strip(log, after):
    return [{k: v for k, v in r.items() if k not in WALL} for r in log if r.get("env_steps", r.get("eval_env_steps", 0)) > after]


def _bc_runs(tmp_path, warm, K):
    from paddlerobotics_b200 import bctrain
    base = _bc_base(tmp_path, warm)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    full = bctrain.main(base + ["--max_steps", str(2 * K * N), "--outdir", a])
    part = bctrain.main(base + ["--max_steps", str(K * N), "--outdir", b])
    return base, full, part, os.path.join(a, "s"), os.path.join(b, "s")


def test_bctrain_warmup_resume_is_bit_for_bit(tmp_path):
    import torch
    from paddlerobotics_b200 import bctrain
    K = 20
    _, full, part, a, b = _bc_runs(tmp_path, True, K)
    assert _strip(part, 0) == _strip(full, 0)[:len(part)] and len(part) == 3              # two uninterrupted runs agree (evaluations at 1, 10, 20 iterations)
    saved = _load(os.path.join(b, "state.pt"))
    assert saved["command"] == "bctrain" and saved["loop"]["total"] == K * N and saved["rpm"]["size"] == K * N
    assert saved["rpm"]["obs"].shape == (K * N, 46)                                      # the ring up to its fill level, not --memory rows
    torch.manual_seed(12345); np.random.seed(12345)
    rest = bctrain.main(["--resume", os.path.join(b, "state.pt"), "--max_steps", str(2 * K * N), "--outdir", os.path.dirname(b)])
    assert rest and _strip(rest, K * N) == _strip(full, K * N)
    _same_bc_outdirs(a, b)


def _same_bc_outdirs(a, b):
    import torch
    fa = sorted(f for f in os.listdir(a) if f.startswith("itr_"))
    assert fa and fa == sorted(f for f in os.listdir(b) if f.startswith("itr_"))
    for f in fa:
        _same(torch.load(os.path.join(a, f)), torch.load(os.path.join(b, f)), f)
    return _same_states(a, b)


def test_bctrain_warmup_resume_in_a_new_process(tmp_path):
    K = 20
    _, full, _, a, b = _bc_runs(tmp_path, True, K)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    out = subprocess.run([sys.executable, "-m", "paddlerobotics_b200.bctrain", "--resume", os.path.join(b, "state.pt"), "--max_steps", str(2 * K * N),
                          "--outdir", os.path.dirname(b)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    rest = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]
    assert rest and _strip(rest, K * N) == _strip(full, K * N)
    _same_bc_outdirs(a, b)


def test_bctrain_learning_resume_takes_the_same_branches(tmp_path):
    """Past the first BC update the learner's f32 atomics make even two uninterrupted runs differ in the last bits (DESIGN §8g), so the
    resumed run must take the same branches: the same records and counters, ring fill, e_step, checkpoints and learner step count."""
    import torch
    from paddlerobotics_b200 import bctrain
    K = 40
    _, full, part, a, b = _bc_runs(tmp_path, False, K)
    assert any("actor_loss" in r for r in part)                                           # the stopped run is past its first update
    torch.manual_seed(12345); np.random.seed(12345)
    rest = bctrain.main(["--resume", os.path.join(b, "state.pt"), "--max_steps", str(2 * K * N), "--outdir", os.path.dirname(b)])
    fa, fb = _strip(full, K * N), _strip(rest, K * N)
    assert fb and len(fa) == len(fb) and any("actor_loss" in r for r in fb)
    for ra, rb in zip(fa, fb):
        assert set(ra) == set(rb)
        for k in ("env_steps", "iters", "rpm_size", "updates", "total_updates", "e_step", "eval_env_steps"):
            assert ra.get(k) == rb.get(k), k
        assert all(np.isfinite(v) for k, v in rb.items() if k.endswith("_loss"))
    sa, sb = _load(os.path.join(a, "state.pt")), _load(os.path.join(b, "state.pt"))
    assert sa["loop"] == sb["loop"] and sa["learner"]["steps"] == sb["learner"]["steps"]
    assert _step(sa["learner"]) == _step(sb["learner"])
    assert (sa["rpm"]["pos"], sa["rpm"]["size"]) == (sb["rpm"]["pos"], sb["rpm"]["size"])
    assert sorted(f for f in os.listdir(a) if f.startswith("itr_")) == sorted(f for f in os.listdir(b) if f.startswith("itr_"))
    assert torch.isfinite(sb["learner"]["snapshot"][1024:-16].view(torch.float32)).all()
