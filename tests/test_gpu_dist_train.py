"""train and pretrain under torchrun with two ranks, against one-rank runs of the same global sizes.  With two or more GPUs the ranks use
NCCL, one GPU each; on one GPU they use gloo and share device 0 (NCCL refuses two ranks on one device).  Each rank of the worker runs
the command in its own directory, so the test sees which ranks wrote files."""
import json
import os
import signal
import socket
import subprocess
import sys
import time

import numpy as np
import pytest

from test_gpu_resume import _same

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT_S = 900

_WORKER = r'''
import json, os, sys
sys.path.insert(0, %r)
from paddlerobotics_b200 import dist_run
cmd, backend, fail = sys.argv[1], sys.argv[2], sys.argv[3] == "1"
argv = sys.argv[4:]
rank, world, local = dist_run.ranks()
os.makedirs("rank%%d" %% rank, exist_ok=True)
os.chdir("rank%%d" %% rank)
import importlib
mod = importlib.import_module("paddlerobotics_b200." + cmd)
learners = []
if cmd == "train":
    make = mod.SACLearner
    mod.SACLearner = lambda *a, **k: learners.append(make(*a, **k)) or learners[-1]
if fail and rank == 1:
    from paddlerobotics_b200 import es
    def take(self, *a, **k):
        raise RuntimeError("rank 1 stops here")
    es.TrainEpisodeStats.take = take
with dist_run.process_group(world, local, backend):
    log = mod.main(argv)
    out = {"rank": rank, "records": len(log)}
    if learners:
        out["replicas_equal"] = dist_run.all_equal(learners[0].replica_state())
    print("WORKER " + json.dumps(out), flush=True)
'''


def _backend():
    import torch
    return "nccl" if torch.cuda.device_count() >= 2 else "gloo"


def _port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _launch(cmd, cwd, timeout=TIMEOUT_S):
    """subprocess.run for a torch.distributed.run launcher, started in a session of its own: on a timeout (or any other exit from here)
    the whole process group, the ranks included, is killed, not the launcher alone."""
    proc = subprocess.Popen(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    finally:
        try:
            os.killpg(proc.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
        proc.wait()
    return subprocess.CompletedProcess(cmd, proc.returncode, out, err)


def _torchrun(tmp, cmd, argv, backend, fail=False):
    """Two ranks of `cmd` in tmp/rank0, tmp/rank1: (completed process, rank 0's JSON records, the WORKER lines)."""
    os.makedirs(tmp, exist_ok=True)
    worker = os.path.join(tmp, "worker.py")
    with open(worker, "w") as f:
        f.write(_WORKER % ROOT)
    out = _launch([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                   "--master-port", str(_port()), worker, cmd, backend, "1" if fail else "0"] + argv + ["--dist_backend", backend], tmp)
    recs, workers = [], []
    for line in out.stdout.splitlines():
        if line.startswith("WORKER "):
            workers.append(json.loads(line[7:]))
        elif line.startswith("{"):
            recs.append(json.loads(line))
    return out, recs, workers


def _ok(out):
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-5000:]


def _same_npz(a, b, keys=None):
    fa = sorted(f for f in os.listdir(a) if f.startswith("itr_") and f.endswith(".npz"))
    assert fa and fa == sorted(f for f in os.listdir(b) if f.startswith("itr_") and f.endswith(".npz"))
    for f in fa:
        with np.load(os.path.join(a, f)) as za, np.load(os.path.join(b, f)) as zb:
            for k in keys or za.files:
                assert za[k].dtype == zb[k].dtype and za[k].tobytes() == zb[k].tobytes(), (f, k)
    return fa


# ---- pretrain: 10 individuals x 2 rollouts, every round evaluates and writes itr_*.npz and state.pt
PRE = ["--popsize", "10", "--es_rollouts", "2", "--es_train_steps", "2", "--task_mode", "ground", "--eval_every_steps", "1", "--suffix", "s",
       "--save_state", "1", "--seed", "3", "--sigma", "0.05"]


def test_pretrain_two_ranks_equal_one_and_resume(tmp_path, capsys):
    import torch
    from paddlerobotics_b200 import pretrain
    one = str(tmp_path / "one")
    full1 = pretrain.main(PRE + ["--max_steps", "30000", "--outdir", one])
    capsys.readouterr()
    ends = [r["env_steps"] for r in full1 if "checkpoint" in r]
    assert len(ends) >= 4, ends
    k = len(ends) // 2
    backend = _backend()
    out, full2, _ = _torchrun(str(tmp_path / "w2"), "pretrain", PRE + ["--max_steps", "30000", "--outdir", "o"], backend)
    _ok(out)
    assert full2 == full1                                                           # every record, bit for bit (JSON floats round-trip)
    a, b = os.path.join(one, "s"), str(tmp_path / "w2" / "rank0" / "o" / "s")
    _same_npz(a, b)
    sa, sb = torch.load(os.path.join(a, "state.pt"), weights_only=False), torch.load(os.path.join(b, "state.pt"), weights_only=False)
    sa.pop("args"); sb.pop("args")
    _same(sa, sb)
    assert os.listdir(tmp_path / "w2" / "rank1") == []                              # only rank 0 writes
    # stopped after k rounds at two ranks, resumed to the end at two ranks: the uninterrupted run
    run = str(tmp_path / "r2")
    out, part, _ = _torchrun(run, "pretrain", PRE + ["--max_steps", str(ends[k - 1]), "--outdir", "o"], backend)
    _ok(out)
    assert part == full1[:len(part)] and sum("checkpoint" in r for r in part) == k
    state = os.path.join(run, "rank0", "o", "s", "state.pt")
    out, rest, _ = _torchrun(run, "pretrain", ["--resume", state, "--max_steps", "30000", "--outdir", "o"], backend)
    _ok(out)
    assert rest == full1[len(part):]
    c = os.path.join(run, "rank0", "o", "s")
    _same_npz(a, c)
    sc = torch.load(os.path.join(c, "state.pt"), weights_only=False)
    sc.pop("args")
    _same(sa, sc)
    assert os.listdir(os.path.join(run, "rank1")) == []


# ---- train: 256 global envs; --act_bound 0 makes the policy's residual zero, so the ES phase (which runs after the warm-up, when the
#      learner has started and the ranks' learners differ from the one-rank learner) depends on the gait and the solver only
N = 256
TRAIN_ES = ["--num_envs", str(N), "--batch", "256", "--memory", "100000", "--warmup_steps", str(2 * N), "--ES", "1", "--popsize", "10",
            "--es_rollouts", "2", "--es_every_steps", str(8 * N), "--es_train_steps", "2", "--e_step", "100", "--act_bound", "0", "--task_mode",
            "ground", "--graph_iter", "0", "--log_every", "5", "--eval_every_steps", str(8 * N), "--max_steps", str(26 * N), "--suffix", "s", "--seed", "3"]


def test_train_es_phase_two_ranks_equal_one(tmp_path, capsys):
    from paddlerobotics_b200 import train
    one = str(tmp_path / "one")
    train.main(TRAIN_ES + ["--outdir", one])
    es1 = [json.loads(l) for l in capsys.readouterr().out.splitlines() if l.startswith('{"ES_gen"')]
    assert len(es1) == 6, es1                                                       # three ES phases of two generations
    out, recs, workers = _torchrun(str(tmp_path / "w2"), "train", TRAIN_ES + ["--outdir", "o"], "gloo")
    _ok(out)
    assert [r for r in recs if "ES_gen" in r] == es1
    _same_npz(os.path.join(one, "s"), str(tmp_path / "w2" / "rank0" / "o" / "s"), keys=("w", "b", "param"))
    assert os.listdir(tmp_path / "w2" / "rank1") == []
    assert sorted(w["rank"] for w in workers) == [0, 1] and all(w["replicas_equal"] for w in workers)


# ---- train with learning on flat ground with the gentle open-loop gait (--act_bound 0): every episode runs to --e_step
E_STEP, LOG_EVERY = 10, 20
TRAIN_LEARN = ["--num_envs", str(N), "--batch", "256", "--warmup_steps", str(4 * N), "--ES", "0", "--task_mode", "ground", "--act_bound", "0",
               "--footheight", "0.03", "--steplen", "0.02", "--e_step", str(E_STEP), "--log_every", str(LOG_EVERY), "--train_eval_envs", "2",
               "--eval_every_steps", str(40 * N), "--max_steps", str(120 * N), "--suffix", "s"]


@pytest.mark.parametrize("graph_iter", [0, 1])
def test_train_learning_two_ranks(tmp_path, graph_iter):
    backend = "gloo" if graph_iter == 0 else "nccl"
    if backend == "nccl" and _backend() != "nccl":
        pytest.skip("the captured iteration at two ranks needs NCCL, which needs two GPUs")
    out, recs, workers = _torchrun(str(tmp_path), "train", TRAIN_LEARN + ["--graph_iter", str(graph_iter), "--outdir", "o"], backend)
    _ok(out)
    assert sorted(w["rank"] for w in workers) == [0, 1]
    assert all(w["replicas_equal"] for w in workers)                                # after the run; train itself checks at every block
    assert [w["records"] for w in sorted(workers, key=lambda w: w["rank"])][1] == 0
    train_recs = [r for r in recs if "train_episodes" in r]
    assert len(train_recs) == 120 // LOG_EVERY
    for r in train_recs:
        assert r["env_steps"] == r["iters"] * N                                     # global env steps
        assert r["train_nonfinite_episodes"] == 0, r
        assert r["train_episode_step"] == E_STEP, r                                 # every episode reached the limit ...
        assert r["train_episodes"] == N * (LOG_EVERY // E_STEP), r                  # ... in every env of both ranks
        if r["critic_loss"] is not None:
            assert np.isfinite([r["critic_loss"], r["actor_loss"]]).all(), r
    assert sum(r["critic_loss"] is not None for r in train_recs) >= 4
    assert len([r for r in recs if "eval_episode_reward" in r]) == 3
    files = sorted(os.listdir(tmp_path / "rank0" / "o" / "s"))
    assert files == sorted("itr_%d.%s" % (k * 40 * N, e) for k in (1, 2, 3) for e in ("pt", "npz"))
    assert os.listdir(tmp_path / "rank1") == []


def test_a_failing_rank_ends_the_run(tmp_path):
    t0 = time.time()
    out, _, _ = _torchrun(str(tmp_path), "train", TRAIN_LEARN + ["--graph_iter", "0", "--max_steps", str(40 * N)], "gloo", fail=True)
    assert out.returncode != 0
    assert "rank 1 stops here" in out.stdout + out.stderr
    assert time.time() - t0 < TIMEOUT_S
    ps = subprocess.run(["ps", "-eo", "args"], capture_output=True, text=True).stdout
    assert str(tmp_path) not in ps, ps                                              # no rank left behind


_CAPTURE_WORKER = r'''
import os, sys
sys.path.insert(0, %r)
import torch
import torch.distributed as dist
from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
assert os.environ["WORLD_SIZE"] == "1"
dev = 0
dist.init_process_group("nccl", device_id=torch.device("cuda", dev))      # a real NCCL group, of the one rank the launcher started
try:
    B, D = 256, 49
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    obs, act, nobs = r(B, D), torch.rand(B, 12, device="cuda", generator=g) * 2 - 1, r(B, D)
    rew, term, e1, e2 = r(B), (torch.rand(B, device="cuda", generator=g) > 0.1).float(), r(B, 12), r(B, 12)
    # the data-parallel path (world > 1: phases with the gradient all-reduces between them) on the one-rank group: every all-reduce is
    # a real NCCL call, and the average over one rank leaves the gradients as they are
    eager, cap = (SACLearner(MujocoAgent(D, 12, device=dev, seed=3), B, world=2) for _ in range(2))
    for L in (eager, cap):
        L.learn(obs, act, rew, nobs, term, eps_next=e1, eps_cur=e2, pull=False)
    flat = lambda L: (L.pull(), torch.cat(flatten_params(L.agent.params)))[1]
    start = cap.replica_state().clone()
    p0 = flat(cap)
    for _ in range(3):
        eager.learn(obs, act, rew, nobs, term, eps_next=e1, eps_cur=e2, pull=False)
    # train's captured iteration: the learner on its own stream inside one CUDA graph, the all-reduces with it
    s_cap, s_learn = torch.cuda.Stream(), torch.cuda.Stream()
    s_cap.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s_cap):
        s_learn.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s_learn):
            cap.learn(obs, act, rew, nobs, term, eps_next=e1, eps_cur=e2, pull=False)
        torch.cuda.current_stream().wait_stream(s_learn)
    torch.cuda.current_stream().wait_stream(s_cap)
    assert torch.equal(cap.replica_state(), start)           # capture records, it does not run
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    fa, fb = flat(eager), flat(cap)
    moved = (fb - p0).abs().max().item()
    diff = (fa - fb).abs().max().item()
    print("CAPTURE moved %%.3e diff %%.3e" %% (moved, diff), flush=True)
    assert moved > 1e-6 and diff <= 1e-3 * moved, (moved, diff)
finally:
    dist.destroy_process_group()
print("CAPTURE ok", flush=True)
'''


def test_nccl_all_reduces_captured_in_the_learner_graph(tmp_path):
    """--graph_iter 1 at W > 1 captures the learner's NCCL all-reduces in the iteration's graph.  Two ranks need two GPUs for NCCL; on
    one GPU this runs the same data-parallel learner on a one-rank NCCL group: three replays of the captured update move the learner as
    three eager updates do (the learner's f32 atomics allow last-bit differences between two runs)."""
    worker = tmp_path / "capture.py"
    worker.write_text(_CAPTURE_WORKER % ROOT)
    out = _launch([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr", "127.0.0.1",
                   "--master-port", str(_port()), str(worker)], str(tmp_path))
    _ok(out)
    assert "CAPTURE ok" in out.stdout, out.stdout[-2000:]
