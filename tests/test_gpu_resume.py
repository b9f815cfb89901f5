"""Stopping and continuing a training run on the GPU: the env snapshot (b2q_snapshot_*), the learner snapshot (b2q_sac_snapshot_*) and
train.py's --save_state / --resume, each checked bit for bit against the run that was never stopped."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(__import__("torch").uint8).cpu()


def _same(a, b, path="state"):
    """Recursive bitwise equality of state dicts (tensors, arrays, scalars, tuples)."""
    import torch
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, path
        assert torch.equal(_bits(a), _bits(b)), path
    elif isinstance(a, np.ndarray):
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), path
    elif isinstance(a, dict):
        assert set(a) == set(b), (path, set(a) ^ set(b))
        for k in a:
            _same(a[k], b[k], "%s.%s" % (path, k))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (path, i))
    else:
        assert a == b or (a != a and b != b), (path, a, b)


def _gait():
    from paddlerobotics_b200.train import etg_prior
    _, w, b, _ = etg_prior()
    return w, b


ENV_CFG = dict(action_filter=1, ring_depth=4, max_episode_steps=25, stuck_termination=1, body_collisions=1)


def _make_env(prec, n=64, task="stairstair", **over):
    from paddlerobotics_b200.env import SENSOR_NOISE_STDDEV, VecQuadrupedalEnv
    from paddlerobotics_b200.etg import dynamic_dict_to_row
    from paddlerobotics_b200.terrain import make_terrain
    cfg = dict(ENV_CFG, noise_stdev=SENSOR_NOISE_STDDEV, noise_seed=11)
    cfg.update(over)
    env = VecQuadrupedalEnv(n, precision=prec, auto_reset=True, heightfield=make_terrain(task), **cfg)
    env.set_dynamics(np.tile(dynamic_dict_to_row({"control_latency": 20}), (n, 1)))      # 20 ms control latency through the observation ring
    return env


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_env_snapshot_continues_bit_for_bit(prec):
    import torch
    w, b = _gait()
    A = _make_env(prec)
    A.reset(w, b)
    g = torch.Generator(device="cuda").manual_seed(0)
    K, M = 40, 40
    acts = (torch.rand(K + M, 64, 12, generator=g, device="cuda", dtype=A.dtype) * 2 - 1) * 0.3
    dones = 0
    for k in range(K):
        dones += int(A.step(acts[k])[2].sum())
    A.set_max_episode_steps(20)                       # a host field: the new handle is created with 25
    sd = A.state_dict()
    B = _make_env(prec)
    B.load_state_dict(sd)
    assert B.cfg.max_episode_steps == 20
    _same(B.state_dict(), sd)
    for k in range(K, K + M):
        oa = [x.clone() for x in A.step(acts[k])]
        ob = B.step(acts[k])
        dones += int(oa[2].sum())
        for x, y, name in zip(oa, ob, ("obs", "reward", "done", "info")):
            assert torch.equal(_bits(x), _bits(y)), (k, name)
        assert torch.equal(_bits(A.get_state()), _bits(B.get_state())), k
    assert dones > 64                                 # auto-reset episodes cross the save point
    A.close(); B.close()


def _load_rc(env, blob):
    import torch
    d = blob.to(env.device)
    rc = env.lib.b2q_snapshot_load(env.h, d.data_ptr(), env._stream())
    torch.cuda.synchronize()
    return rc, env.lib.b2q_last_error(env.h).decode()


def test_env_snapshot_refusals():
    import torch
    A = _make_env("f32")
    blob = A.state_dict()["snapshot"]
    for kw, field in ((dict(n=32), "size"), (dict(prec="f64"), "size"), (dict(sensor_imu=2), "obs_dim"), (dict(task="ground"), "terrain_type"),
                      (dict(noise_seed=12), "noise_seed"), (dict(action_filter=0), "action_filter")):
        kw = dict(kw)
        B = _make_env(kw.pop("prec", "f32"), **kw)
        want = int(B.lib.b2q_snapshot_bytes(B.h))
        if want == blob.numel():
            rc, err = _load_rc(B, blob)
            assert rc == -1 and field in err, (kw, err)
        else:
            with pytest.raises(ValueError):
                B.load_state_dict(A.state_dict())
            big = torch.zeros(max(want, blob.numel()), dtype=torch.uint8)
            big[:blob.numel()] = blob
            rc, err = _load_rc(B, big)                 # the header alone refuses it
            assert rc == -1, (kw, err)
        B.close()
    from paddlerobotics_b200.env import SENSOR_NOISE_STDDEV, VecQuadrupedalEnv
    from paddlerobotics_b200.terrain import make_terrain
    hf, x0, y0, cell = make_terrain("stairstair")
    D = VecQuadrupedalEnv(64, auto_reset=True, heightfield=(hf + 0.01, x0, y0, cell), noise_stdev=SENSOR_NOISE_STDDEV, noise_seed=11, **ENV_CFG)
    rc, err = _load_rc(D, blob)
    assert rc == -1 and "height field" in err, err
    D.close()
    bad = blob.clone(); bad[0] ^= 1
    rc, err = _load_rc(A, bad)
    assert rc == -1 and "magic" in err
    trunc = blob.clone(); trunc[16:24] = torch.tensor([blob.numel() - 64], dtype=torch.int64).view(torch.uint8)   # header's total size
    rc, err = _load_rc(A, trunc)
    assert rc == -1 and "size" in err
    with pytest.raises(ValueError):
        A.load_state_dict(dict(A.state_dict(), snapshot=blob[:-16]))
    A.close()


def test_learner_snapshot_next_learn_is_bit_identical():
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    g = torch.Generator(device="cuda").manual_seed(3)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")
    B, D = 128, 49
    batch = (r(B, D), r(B, 12).clamp(-1, 1), r(B), r(B, D), (torch.rand(B, generator=g, device="cuda") > 0.1).float())
    L1 = SACLearner(MujocoAgent(D, 12, seed=0), B)
    for _ in range(3):
        L1.learn(*batch, pull=False)
    sd = L1.state_dict()
    # layout: header, actor, critic, target, Adam m/v of the actor and of the critics, 4 loss floats, then d_step (step count, ticket) in 16 bytes
    na, nc = L1.na, L1.nc
    assert sd["snapshot"].numel() == 1024 + 4 * (3 * na + 4 * nc + 4) + 16
    assert _step(sd) == [3, 0]
    L1.pull()
    from paddlerobotics_b200.agent import flatten_params
    fa, fc = flatten_params(L1.agent.params)
    payload = sd["snapshot"][1024:-16].view(torch.float32)
    assert torch.equal(payload[:na], fa.cpu()) and torch.equal(payload[na:na + nc], fc.cpu())
    L2 = SACLearner(MujocoAgent(D, 12, seed=1), B)
    L2.load_state_dict(sd)
    _same(L2.state_dict(), sd)
    assert torch.equal(L2.agent.params["actor_model.l1.weight"], L1.agent.params["actor_model.l1.weight"])    # load_state_dict pulls
    obs = r(256, D)
    for mode in (0, 1):                                # the forward has no atomics: bit for bit
        a1 = L1.actor.forward(obs, mode=mode, seed=9)[0].clone()
        a2 = L2.actor.forward(obs, mode=mode, seed=9)[0].clone()
        assert torch.equal(_bits(a1), _bits(a2)), mode
    # A learn is not bit-reproducible even on one learner: the split-K GEMMs and the loss sums add with f32 atomics in run-dependent order.
    # So the next learn of the loaded learner is held to the spread of two learners loaded from the same blob.
    L3 = SACLearner(MujocoAgent(D, 12, seed=2), B)
    L3.load_state_dict(sd)
    outs = [(L.learn(*batch, pull=False).clone(), L.state_dict()) for L in (L1, L2, L3)]
    for (l, st) in outs[1:]:
        assert torch.allclose(l, outs[0][0], rtol=1e-5, atol=1e-6)
        assert st["steps"] == outs[0][1]["steps"]
        a, b = st["snapshot"][1024:].view(torch.float32)[:-4], outs[0][1]["snapshot"][1024:].view(torch.float32)[:-4]
        assert float((a - b).abs().max()) < 2e-5       # parameters, target, moments, losses (test_gpu_sac's split-K bound)
        assert torch.equal(st["snapshot"][-16:], outs[0][1]["snapshot"][-16:])    # device step counter and ticket
    assert _step(outs[0][1]) == [4, 0]
    L3.close()
    for kw, field in ((dict(batch=256), "batch"), (dict(actor_lr=1e-3), "actor_lr"), (dict(obs_dim=46), "obs_dim")):
        od = kw.pop("obs_dim", D)
        L3 = SACLearner(MujocoAgent(od, 12), kw.pop("batch", B), **kw)
        blob = sd["snapshot"].to("cuda")
        if int(L3.lib.b2q_sac_snapshot_bytes(L3.h)) == blob.numel():
            assert L3.lib.b2q_sac_snapshot_load(L3.h, blob.data_ptr(), L3._stream()) == -1
            assert field in L3.lib.b2q_sac_last_error(L3.h).decode()
        else:
            with pytest.raises(ValueError):
                L3.load_state_dict(sd)
        L3.close()
    L1.close(); L2.close()


# ---- train.main: uninterrupted 2K iterations against K iterations + --resume to 2K
N = 64
BASE = ["--num_envs", str(N), "--batch", "128", "--memory", "20000", "--warmup_steps", str(10 * N), "--log_every", "5", "--ES", "0",
        "--task_mode", "ground", "--eval_every_steps", str(10 * N), "--suffix", "s", "--save_state", "1"]
WALL = ("env_steps_per_s", "interval_env_steps_per_s")
# Only warm-up is bit-reproducible end to end: from the first learn on, the learner's f32 atomics make even two uninterrupted runs differ
# in the last bits, and the envs amplify that.  The "warmup_only" case stays in warm-up and must match bit for bit; the others must take
# the same branches (iterations, log cadence, ES phases, graph capture, e_step, replay cursor) and stay finite.
CASES = {
    "warmup_only": (["--graph_iter", "1", "--warmup_steps", str(30 * N)], 10),
    "eager": (["--graph_iter", "0"], 30),
    "graph": (["--graph_iter", "1"], 30),
    "warmup": (["--graph_iter", "1", "--warmup_steps", str(30 * N)], 20),
    "es_rpm": (["--graph_iter", "1", "--ES", "1", "--popsize", "10", "--es_rollouts", "1", "--es_every_steps", str(31 * N), "--es_train_steps", "2",
                "--es_rpm", "1", "--e_step", "30"], 30),
    "es_twice": (["--graph_iter", "1", "--ES", "1", "--popsize", "10", "--es_rollouts", "1", "--es_every_steps", str(15 * N), "--es_train_steps", "2",
                  "--es_rpm", "1", "--e_step", "30"], 30),
    "e_step_growth": (["--graph_iter", "1", "--e_step_growth", "50", "--e_step", "20"], 30),
    "sensor_noise": (["--graph_iter", "1", "--sensor_noise", "1", "--seed", "4", "--task_mode", "stairstair"], 30),
}


def _step(learner_sd):
    """The learner's device step counter and closing-Adam ticket from a SACLearner.state_dict()."""
    return learner_sd["snapshot"][-16:-8].view(__import__("torch").int32).tolist()


def _strip(log, after):
    return [{k: v for k, v in r.items() if k not in WALL} for r in log if r.get("env_steps", 0) > after]


def _compare_outdirs(a, b, after):
    import torch
    sa, sb = torch.load(os.path.join(a, "state.pt"), weights_only=False), torch.load(os.path.join(b, "state.pt"), weights_only=False)
    sa.pop("args"); sb.pop("args")
    _same(sa, sb)
    fa = sorted(f for f in os.listdir(a) if f.startswith("itr_") and int(f.split("_")[1].split(".")[0]) > after)
    fb = sorted(f for f in os.listdir(b) if f.startswith("itr_") and int(f.split("_")[1].split(".")[0]) > after)
    assert fa == fb and fa
    for f in fa:
        if f.endswith(".pt"):
            _same(torch.load(os.path.join(a, f)), torch.load(os.path.join(b, f)), f)
        else:
            with np.load(os.path.join(a, f)) as za, np.load(os.path.join(b, f)) as zb:
                assert sorted(za.files) == sorted(zb.files)
                for k in za.files:
                    assert za[k].tobytes() == zb[k].tobytes(), (f, k)
    return sa


@pytest.mark.parametrize("case", sorted(CASES))
def test_resumed_training_equals_the_uninterrupted_run(tmp_path, case):
    import torch
    from paddlerobotics_b200 import train
    extra, K = CASES[case]
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    full = train.main(BASE + extra + ["--max_steps", str(2 * K * N), "--outdir", a])
    train.main(BASE + extra + ["--max_steps", str(K * N), "--outdir", b])
    saved = torch.load(os.path.join(b, "s", "state.pt"), weights_only=False)
    assert saved["loop"]["total"] == K * N
    if case == "warmup":
        assert saved["rpm"]["size"] < 30 * N and not saved["graph"]
    if case == "graph":
        assert saved["graph"]
    if case == "e_step_growth":
        assert not saved["graph"] and saved["loop"]["e_step"] > 20
    if case == "es_rpm":                                 # the save point is the iteration before the ES phase
        assert saved["solver"]["attrs"]["first_iteration"] and saved["loop"]["last_es"] == 0
    if case == "es_twice":                               # ES phases at iterations 15 and 30, the save after the second, two more after the resume
        assert saved["loop"]["last_es"] == K * N and saved["solver"]["attrs"]["sigma"] < 0.02
    torch.manual_seed(12345); np.random.seed(12345)     # the state must bring back both generators
    rest = train.main(["--resume", os.path.join(b, "s", "state.pt"), "--max_steps", str(2 * K * N), "--outdir", b])
    _check(full, rest, os.path.join(a, "s"), os.path.join(b, "s"), K * N, exact=case == "warmup_only", es_rows=case.startswith("es_"))


def _check(full, rest, a, b, after, exact, es_rows=False):
    """exact: the whole final state, the itr_* files and the log records after `after` are identical.  Otherwise the two runs must take the same
    branches: the same log records and keys, loop counters, graph mode, host and device learner step counts, replay samples drawn, checkpoints,
    and the parts of the ES solver that fitness values do not decide (sigma after its decays, NumPy's RNG state, first_iteration).  es_rows:
    the ES phase appends rows up to each rollout's first done, which a last-bit difference of the policy can move, so the replay's position
    and fill level are not compared."""
    import torch
    fa, fb = _strip(full, after), _strip(rest, after)
    assert fb and [r["env_steps"] for r in fa] == [r["env_steps"] for r in fb]
    if exact:
        assert fa == fb
        _compare_outdirs(a, b, after)
        return
    for ra, rb in zip(fa, fb):
        assert set(ra) == set(rb)
        assert all((ra[k] is None) == (rb[k] is None) for k in ra)
    sa, sb = torch.load(os.path.join(a, "state.pt"), weights_only=False), torch.load(os.path.join(b, "state.pt"), weights_only=False)
    assert sa["loop"] == sb["loop"] and sa["graph"] == sb["graph"] and sa["learner"]["steps"] == sb["learner"]["steps"]
    assert _step(sa["learner"]) == _step(sb["learner"]) and _step(sa["learner"])[1] == 0
    assert sa["rpm"]["samples"] == sb["rpm"]["samples"]
    if sa["rpm"]["cursor"] is not None:
        assert int(sa["rpm"]["cursor"][2]) == int(sb["rpm"]["cursor"][2])
    if not es_rows:
        assert (sa["rpm"]["pos"], sa["rpm"]["size"]) == (sb["rpm"]["pos"], sb["rpm"]["size"])
        assert sa["rpm"]["cursor"] is None or torch.equal(sa["rpm"]["cursor"], sb["rpm"]["cursor"])
    ga, gb = sa["solver"], sb["solver"]
    assert ga["attrs"]["sigma"] == gb["attrs"]["sigma"] and ga["attrs"]["first_iteration"] == gb["attrs"]["first_iteration"]
    _same(ga["np_random"], gb["np_random"], "np_random")
    assert sorted(f for f in os.listdir(a) if f.startswith("itr_")) == sorted(f for f in os.listdir(b) if f.startswith("itr_"))
    assert torch.isfinite(sb["learner"]["snapshot"][1024:-16].view(torch.float32)).all()


def test_resume_in_a_new_process(tmp_path):
    from paddlerobotics_b200 import train
    extra, K = CASES["warmup_only"]
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    full = train.main(BASE + extra + ["--max_steps", str(2 * K * N), "--outdir", a])
    train.main(BASE + extra + ["--max_steps", str(K * N), "--outdir", b])
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    out = subprocess.run([sys.executable, "-m", "paddlerobotics_b200.train", "--resume", os.path.join(b, "s", "state.pt"), "--max_steps", str(2 * K * N),
                          "--outdir", b], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    rest = [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{") and '"env_steps_per_s"' in l]
    _check(full, rest, os.path.join(a, "s"), os.path.join(b, "s"), K * N, exact=True)
