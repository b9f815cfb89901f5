"""ETG pretraining on the GPU: the fused episode-statistics kernel (b2q_es_accumulate_terms) against b2q_es_accumulate and a NumPy
restatement, PopulationEvaluator.evaluate(terms=) against the float64 oracle, the pretrain command end to end (fitness bit for bit against
the evaluator, determinism, checkpoints), the round trip into train.py --ETG_path, the shared evaluation loop against the loop it
replaced, and the env_test gait-table export."""
import ctypes as C
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SHIPPED = os.path.join(ROOT, "paddlerobotics_b200", "data", "etg_shipped_gait.npz")


def _np(t):
    return t.double().cpu().numpy()


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cols(cols):
    return (C.c_int32 * max(16, len(cols)))(*cols)


# ---------------------------------------------------------------------------------------------------------------- 1. the kernel

def _accumulate_terms(lib, reward, done, alive, ret, length, info, cols, term_sum, count_col, thresh, count, n, es):
    p = lambda t: None if t is None else t.data_ptr()
    return lib.b2q_es_accumulate_terms(p(reward), p(done), p(alive), p(ret), p(length), p(info), 56, _cols(cols), len(cols), p(term_sum), count_col,
                                       thresh, p(count), n, es, _stream())


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("n", [1, 1000])
def test_accumulate_terms_kernel(precision, n):
    """60 steps of random rewards, info rows and done patterns: ret / len / alive equal b2q_es_accumulate bit for bit; the term sums and
    counts equal a NumPy restatement that adds in the same order and dtype; a NaN term propagates, a NaN velx does not count and a velx
    exactly at the threshold does."""
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import INFO
    lib = _lib.load()
    dt, npdt = (torch.float32, np.float32) if precision == "f32" else (torch.float64, np.float64)
    es = 4 if precision == "f32" else 8
    rng = np.random.default_rng(n)
    T, thresh = 60, 0.3
    cols = [INFO[k] for k in ("torso", "feet", "up", "tau", "badfoot", "footcontact")] + [INFO["step"], INFO["torso"]]   # a repeated column too
    rew = rng.normal(size=(T, n)).astype(npdt)
    info = rng.uniform(-1, 1, (T, n, 56)).astype(npdt)
    info[:, :, 0] = rng.choice(np.array([0.1, 0.3, 0.5], dtype=npdt), (T, n))            # velx below, AT and above the threshold
    done = (rng.random((T, n)) < 0.04).astype(np.uint8)
    info[0, 0, cols[1]] = np.nan                                                          # env 0 is alive at step 0: its feet sum is NaN
    info[1, 0, 0] = np.nan                                                                # a NaN velx never counts
    dev = lambda a: torch.as_tensor(a, device="cuda")
    ref_alive, ref_ret, ref_len = dev(np.ones(n, np.uint8)), torch.zeros(n, dtype=dt, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    alive, ret, length = ref_alive.clone(), ref_ret.clone(), ref_len.clone()
    tsum, count = torch.zeros(len(cols), n, dtype=dt, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    np_alive, np_ts, np_cnt = np.ones(n, bool), np.zeros((len(cols), n), npdt), np.zeros(n, np.int32)
    for t in range(T):
        r, d, inf = dev(rew[t]), dev(done[t]), dev(info[t])
        assert lib.b2q_es_accumulate(r.data_ptr(), d.data_ptr(), ref_alive.data_ptr(), ref_ret.data_ptr(), ref_len.data_ptr(), n, es, _stream()) == 0
        assert _accumulate_terms(lib, r, d, alive, ret, length, inf, cols, tsum, 0, thresh, count, n, es) == 0
        m = np_alive.copy()
        for j, c in enumerate(cols):
            np_ts[j, m] = np_ts[j, m] + info[t, m, c]
        np_cnt[m] += (info[t, m, 0] >= npdt(thresh)).astype(np.int32)
        np_alive &= ~done[t].astype(bool)
    torch.cuda.synchronize()
    assert torch.equal(ret, ref_ret) and torch.equal(length, ref_len) and torch.equal(alive, ref_alive)
    got = tsum.cpu().numpy()
    assert np.array_equal(got, np_ts, equal_nan=True) and got.dtype == npdt
    assert np.array_equal(count.cpu().numpy(), np_cnt)
    assert np.isnan(got[1, 0]) and np.isfinite(got[0, 0])
    assert np.array_equal(got[0], got[len(cols) - 1])                                     # the repeated column
    # velx exactly at the threshold counts; NaN does not (env 0: velx at step 1 is NaN and was not counted)
    one = dev(np.array([1], np.uint8))
    a1, r1, l1, c1 = dev(np.ones(1, np.uint8)), torch.zeros(1, dtype=dt, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    for v in (thresh, np.nextafter(npdt(thresh), npdt(0)), np.nan):
        row = torch.zeros(1, 56, dtype=dt, device="cuda"); row[0, 0] = float(npdt(v))
        assert _accumulate_terms(lib, torch.zeros(1, dtype=dt, device="cuda"), one * 0, a1, r1, l1, row, [], None, 0, thresh, c1, 1, es) == 0
    torch.cuda.synchronize()
    assert int(c1) == 1 and int(l1) == 3


def test_accumulate_terms_edges_and_invalid_arguments():
    """ncols = 0 with a NULL count (count_col = -1) is the plain accumulator; every invalid argument returns -1 and touches nothing."""
    import torch
    from paddlerobotics_b200 import _lib
    lib = _lib.load()
    n = 300                                                                               # a partial last block
    rew, done = torch.randn(n, device="cuda"), (torch.rand(n, device="cuda") < 0.5).to(torch.uint8)
    a, r, l = torch.ones(n, dtype=torch.uint8, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    a2, r2, l2 = a.clone(), r.clone(), l.clone()
    assert _accumulate_terms(lib, rew, done, a, r, l, None, [], None, -1, 0.3, None, n, 4) == 0
    assert lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), a2.data_ptr(), r2.data_ptr(), l2.data_ptr(), n, 4, _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(a, a2) and torch.equal(r, r2) and torch.equal(l, l2)
    info, ts, cnt = torch.zeros(n, 56, device="cuda"), torch.zeros(2, n, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    good = dict(reward=rew, done=done, alive=a, ret=r, length=l, info=info, cols=[1, 2], term_sum=ts, count_col=0, thresh=0.3, count=cnt, n=n, es=4)
    assert _accumulate_terms(lib, **good) == 0
    bad = [dict(reward=None), dict(done=None), dict(alive=None), dict(ret=None), dict(length=None), dict(info=None), dict(term_sum=None),
           dict(count=None), dict(cols=[1, 56]), dict(cols=[-1]), dict(cols=list(range(17))), dict(count_col=56), dict(count_col=-2),
           dict(n=0), dict(es=2), dict(cols=[], term_sum=None, info=None)]
    before = [t.clone() for t in (a, r, l, ts, cnt)]
    for b in bad:
        assert _accumulate_terms(lib, **{**good, **b}) == -1, b
    assert lib.b2q_es_accumulate_terms(rew.data_ptr(), done.data_ptr(), a.data_ptr(), r.data_ptr(), l.data_ptr(), info.data_ptr(), 56, None, 2,
                                       ts.data_ptr(), -1, 0.3, None, n, 4, _stream()) == -1     # NULL cols with ncols > 0
    assert lib.b2q_es_accumulate_terms(rew.data_ptr(), done.data_ptr(), a.data_ptr(), r.data_ptr(), l.data_ptr(), info.data_ptr(), 0, _cols([1]), 1,
                                       ts.data_ptr(), -1, 0.3, None, n, 4, _stream()) == -1     # info_dim < 1
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(before, (a, r, l, ts, cnt)))


def test_accumulate_terms_in_a_cuda_graph():
    """The column array travels in the kernel arguments: the call captures and replays."""
    import torch
    from paddlerobotics_b200.es import EpisodeStats
    from paddlerobotics_b200 import _lib
    n = 64
    rew, done, info = torch.ones(n, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.rand(n, 56, device="cuda")
    st = EpisodeStats(_lib.load(), n, torch.float32, torch.device("cuda"), ("torso", "up"))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        st.step(rew, done, info, C.c_void_p(s.cuda_stream))
    torch.cuda.current_stream().wait_stream(s)
    st.zero()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(st.len, torch.full((n,), 3, dtype=torch.int32, device="cuda"))
    assert torch.allclose(st.term_sum[1], 3 * info[:, 3])


# ---------------------------------------------------------------------------------------------------------------- 2. the evaluator

def test_evaluator_terms_vs_oracle(golden):
    """evaluate(terms=): fitness and length bit-identical to the call without terms; in f64 with residual noise the per-individual term
    means and success rates equal serial float64-oracle rollouts (the tolerance of test_es_population_fitness_vs_oracle)."""
    import torch
    from oracle import oracle as O
    from paddlerobotics_b200._config import INFO
    from paddlerobotics_b200.es import PopulationEvaluator, SimpleGA, solutions_to_etg
    from paddlerobotics_b200.etg import shipped_gait
    from paddlerobotics_b200.train import EVAL_TERMS
    np.random.seed(0)
    ga = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.25, weight_decay=0.005, popsize=4, param=np.zeros(12))
    w, b = solutions_to_etg(ga.ask(), golden["opt_points"], golden["opt_w0"], golden["opt_b0"])
    w[0], b[0] = shipped_gait()                                            # individual 0 walks at ~0.48 m/s: its steps count towards success
    pop, rollouts, T = 4, 2, 45
    ev = PopulationEvaluator(pop, rollouts, max_steps=T, precision="f64")
    scale = np.repeat([0.02, 0.3, 0.3, 0.3], rollouts)[None, :, None]
    noise = torch.tensor(np.random.default_rng(0).uniform(-1, 1, (T, pop * rollouts, 12)) * scale, device="cuda")
    fit0, len0 = [x.clone() for x in ev.evaluate(w, b, residual_noise=noise)]
    fit, mlen, tmean, succ = ev.evaluate(w, b, residual_noise=noise, terms=EVAL_TERMS)
    assert torch.equal(fit, fit0) and torch.equal(mlen, len0)
    assert tuple(tmean.shape) == (len(EVAL_TERMS), pop) and tuple(succ.shape) == (pop,)
    ref_t, ref_s, lens, noise_np = np.zeros((len(EVAL_TERMS), pop)), np.zeros(pop), [], noise.cpu().numpy()
    for i in range(pop):
        for r in range(rollouts):
            o = O.OracleEnv(); o.reset(w[i], b[i])
            sums, cnt = np.zeros(len(EVAL_TERMS)), 0
            for k in range(T):
                _, rew, done, info = o.step(noise_np[k, i * rollouts + r])
                sums += [info[INFO[t]] for t in EVAL_TERMS]
                cnt += info[INFO["velx"]] >= 0.3
                if done:
                    break
            lens.append(k + 1)
            ref_t[:, i] += sums / rollouts; ref_s[i] += cnt / (k + 1) / rollouts
    assert np.abs(_np(tmean) - ref_t).max() < 1e-6, (_np(tmean), ref_t)
    assert np.abs(_np(succ) - ref_s).max() < 1e-12
    assert min(lens) < T and 0 < ref_s.max()                               # some episodes froze early; some steps counted
    ev.env.close()


# ---------------------------------------------------------------------------------------------------------------- 3-4. the command

PRE = ["--popsize", "10", "--es_train_steps", "2", "--task_mode", "ground", "--max_steps", "1", "--eval_every_steps", "1000", "--suffix", "s"]


def _lines(capsys):
    return [l for l in capsys.readouterr().out.splitlines() if l.startswith("{")]


@pytest.fixture(scope="module")
def pretrained(tmp_path_factory):
    """Two identically seeded runs of the command; returns (log, printed lines, files) of each and the first run's outdir."""
    import contextlib
    import io
    from paddlerobotics_b200 import pretrain
    runs = []
    for k in range(2):
        out = str(tmp_path_factory.mktemp("pre%d" % k))
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            log = pretrain.main(PRE + ["--outdir", out])
        d = os.path.join(out, "s")
        files = {f: dict(np.load(os.path.join(d, f))) for f in sorted(os.listdir(d))}
        runs.append((log, [l for l in buf.getvalue().splitlines() if l.startswith("{")], files, d))
    return runs


def test_pretrain_fields_and_fitness_bit_for_bit(pretrained):
    """Every generation line has its fields, and its statistics are those of PopulationEvaluator.evaluate (without terms) on the solutions
    of an identically seeded SimpleGA, bit for bit."""
    from paddlerobotics_b200 import pretrain
    from paddlerobotics_b200.es import PopulationEvaluator, SimpleGA, solutions_to_etg_device
    from paddlerobotics_b200.train import EVAL_TERMS, etg_prior
    log = pretrained[0][0]
    gens = [r for r in log if "ES_step" in r]
    assert len(gens) == 2
    keys = {"fitness_max", "fitness_mean", "fitness_min", "fitness_std", "mean_len", "sigma", "success_rate", "env_steps", "best_reward"}
    keys |= {p + t for t in EVAL_TERMS for p in ("episode_", "mean_")}
    for r in gens:
        assert keys <= set(r), keys - set(r)
        assert 0 <= r["success_rate"] <= 1 and 1 <= r["mean_len"] <= 401
        assert r["mean_torso"] == pytest.approx(r["episode_torso"] / r["mean_len"])
    args = pretrain.parser().parse_args(PRE)
    np.random.seed(0)
    _, w0, b0, prior = etg_prior()
    ga = SimpleGA(12, sigma_init=0.02, sigma_decay=0.99, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize=10, param=np.zeros(12))
    ev = PopulationEvaluator(10, 1, max_steps=401, policy=None, **pretrain.env_config(args))
    steps = 0
    for r in gens:
        sol = ga.ask()
        ws, bs = solutions_to_etg_device(sol, prior, w0, b0)
        fit, mlen = ev.evaluate(ws.cpu().numpy(), bs.cpu().numpy())
        steps += int(ev.len.sum())
        fit = np.where(np.isfinite(_np(fit)), _np(fit), -1e9)
        assert (r["fitness_max"], r["fitness_mean"], r["fitness_min"], r["fitness_std"]) == (float(fit.max()), float(fit.mean()), float(fit.min()), float(np.std(fit)))
        assert r["mean_len"] == float(_np(mlen).mean()) and r["env_steps"] == steps
        ga.tell(fit)
        assert r["sigma"] == float(np.mean(ga.result()[3]))
    ev.env.close()


def test_pretrain_is_deterministic_and_writes_checkpoints(pretrained):
    """A second run with the same seed prints identical lines and writes identical files; itr_*.npz holds w [3,20], b [3], param [12] with
    (w, b) the host fit of prior + param."""
    from paddlerobotics_b200.etg import Opt_with_points
    from paddlerobotics_b200.train import etg_prior
    (log, lines, files, d), (_, lines2, files2, _) = pretrained
    assert lines == lines2 and len(lines) == 3
    assert list(files) == list(files2) and len(files) == 1
    for f in files:
        assert all(np.array_equal(files[f][k], files2[f][k]) for k in files[f])
    (name, z), = files.items()
    ev = [r for r in log if "checkpoint" in r]
    assert len(ev) == 1 and ev[0]["checkpoint"] == name == "itr_%d.npz" % log[1]["env_steps"]
    assert z["w"].shape == (3, 20) and z["b"].shape == (3,) and z["param"].shape == (12,)
    layer, w0, b0, prior = etg_prior()
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, w0=w0, b0=b0, points=prior + z["param"].reshape(-1, 2))
    assert np.array_equal(z["w"], w) and np.array_equal(z["b"], b)
    assert 1 <= ev[0]["eval_length"] <= 601


def test_train_etg_path_round_trip(pretrained, monkeypatch, capsys):
    """train.py --ETG_path <pretrained itr>.npz: the ES solver starts at its param and the first reset uses Opt_with_points(prior + param)."""
    from paddlerobotics_b200 import train
    (_, _, files, d) = pretrained[0]
    path = os.path.join(d, next(iter(files)))
    param = np.load(path)["param"]
    seeds, resets = [], []

    class GA(train.SimpleGA):
        def __init__(self, *a, **k):
            seeds.append(np.array(k["param"]))
            super().__init__(*a, **k)

    class Env(train.VecQuadrupedalEnv):
        def reset(self, ETG_w=None, ETG_b=None, **k):
            resets.append((np.array(ETG_w), np.array(ETG_b)))
            return super().reset(ETG_w, ETG_b, **k)
    monkeypatch.setattr(train, "SimpleGA", GA)
    monkeypatch.setattr(train, "VecQuadrupedalEnv", Env)
    train.main(["--ETG_path", path, "--num_envs", "256", "--batch", "256", "--warmup_steps", "1024", "--log_every", "5", "--max_steps", "2560",
                "--es_every_steps", "1280", "--es_train_steps", "1", "--popsize", "10", "--es_rollouts", "1", "--e_step", "100", "--task_mode", "ground"])
    assert len(seeds) == 1 and np.array_equal(seeds[0], param)
    _, w, b = train.initial_etg(train.parser().parse_args(["--ETG_path", path]))
    assert np.array_equal(resets[0][0], w) and np.array_equal(resets[0][1], b)
    assert any("ES_gen" in json.loads(l) for l in _lines(capsys))


# ---------------------------------------------------------------------------------------------------------------- 5. evaluation

def test_pretrain_eval_writes_frames(pretrained, tmp_path, capsys):
    from paddlerobotics_b200 import pretrain
    (_, _, files, d) = pretrained[0]
    frames = tmp_path / "frames"
    rec = pretrain.main(["--eval", "1", "--load", os.path.join(d, next(iter(files))), "--eval_envs", "4", "--task_mode", "ground",
                         "--render_dir", str(frames), "--render_width", "48", "--render_height", "32"])
    lines = _lines(capsys)
    assert len(lines) == 1 and json.loads(lines[0]) == rec
    assert {"mean_return", "mean_length", "terms", "success_rate"} <= set(rec) and rec["eval_envs"] == 4
    n = len(list(frames.iterdir()))
    assert n == rec["mean_length"] and 1 <= n <= 601                      # four identical envs: every step taken has its frame
    assert sorted(frames.iterdir())[0].name.startswith("img") and (frames / ("img%d.png" % n)).exists()


def _old_eval_loop(args, env_cfg):
    """train.evaluate as it was before the fused kernel: per-term copies of `alive`, 1 + 6 b2q_es_accumulate launches per step."""
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import INFO
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv, apply_dynamic_param
    from paddlerobotics_b200.train import EVAL_MAX_STEP, EVAL_TERMS
    agent = MujocoAgent(49, 12, seed=args.seed)
    agent.restore(args.load)
    z = np.load(args.load[:-3] + ".npz")
    w, b = z["w"], z["b"]
    n = args.eval_envs
    env = apply_dynamic_param(VecQuadrupedalEnv(n, auto_reset=False, **env_cfg), args.dynamic_param)
    lib, dev, es, stream = _lib.load(), env.device, env.obs.element_size(), env._stream()
    nt = len(EVAL_TERMS)
    cols = torch.tensor([INFO[k] for k in EVAL_TERMS], device=dev)
    alive = torch.ones(n, dtype=torch.uint8, device=dev)
    ret, length = torch.zeros(n, dtype=env.dtype, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    t_alive, t_sum, t_len = torch.empty(nt, n, dtype=torch.uint8, device=dev), torch.zeros(nt, n, dtype=env.dtype, device=dev), torch.zeros(nt, n, dtype=torch.int32, device=dev)
    t_val = torch.empty(nt, n, dtype=env.dtype, device=dev)
    obs = env.reset(w, b)
    for steps in range(1, EVAL_MAX_STEP + 2):
        act = agent.predict_batch(obs)
        obs, rew, done, info = env.step(act * args.act_bound, donef=steps > EVAL_MAX_STEP)
        t_val.copy_(info.index_select(1, cols).T)
        t_alive.copy_(alive.expand(nt, n))
        for j in range(nt):
            assert lib.b2q_es_accumulate(t_val[j].data_ptr(), done.data_ptr(), t_alive[j].data_ptr(), t_sum[j].data_ptr(), t_len[j].data_ptr(), n, es, stream) == 0
        assert lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), alive.data_ptr(), ret.data_ptr(), length.data_ptr(), n, es, stream) == 0
        if not bool(alive.any()):
            break
    rec = {"eval_envs": n, "mean_return": float(ret.double().mean()), "mean_length": float(length.double().mean()),
           "terms": {k: float(t_sum[j].double().mean()) for j, k in enumerate(EVAL_TERMS)}}
    env.close()
    return rec


@pytest.mark.parametrize("task", ["stairstair", "ground"])
def test_train_eval_equals_the_old_loop(task, tmp_path, capsys):
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.train import etg_prior
    MujocoAgent(49, 12, seed=5).save(str(tmp_path / "itr_0.pt"))
    _, w, b, _ = etg_prior()
    np.savez(str(tmp_path / "itr_0.npz"), w=w, b=b, param=np.zeros(12))
    argv = ["--eval", "1", "--load", str(tmp_path / "itr_0.pt"), "--task_mode", task, "--eval_envs", "16"]
    rec = train.main(argv)
    args = train.parser().parse_args(argv)
    assert rec == _old_eval_loop(args, train.env_config(args))
    assert set(rec) == {"eval_envs", "mean_return", "mean_length", "terms"}


# ---------------------------------------------------------------------------------------------------------------- 6. export

def test_env_test_exports_the_shipped_gait(tmp_path, monkeypatch):
    from paddlerobotics_b200 import env_test
    monkeypatch.chdir(tmp_path)
    table = env_test.main(["--load", SHIPPED, "--save", "1"])
    saved = np.load(str(tmp_path / "gait_action_list_ETG_exp.npy"))
    golden = np.load(os.path.join(GOLDEN, "gait_action_list_ETG_exp.npy"))
    assert saved.shape == (600, 12) and np.array_equal(saved, table)
    assert np.abs(saved - golden).max() < 2e-6
