"""Per-episode training statistics on the GPU (b2q_train_episode_stats, es.TrainEpisodeStats) and the batched train.py that logs them: the
kernel bit for bit against a NumPy float64 restatement in the same addition order, against episodes cut on the host from a real auto-reset
rollout, and train.main end to end (the new log keys, the evaluation block and what it must leave alone, the graph recapture after an
e_step growth, --ETG_T reaching the kernel, and the observation widths of the --sensor_* flags)."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TERMS16 = ("velx", "torso", "feet", "up", "tau", "stand", "badfoot", "footcontact", "done", "nan", "energy", "base_z", "fall", "step", "torso", "up")


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class RefStats:
    """The kernel's arithmetic in NumPy float64, one vectorised operation per kernel statement (elementwise: the same order per env)."""

    def __init__(self, n, cols, count_col, thresh=0.3):
        self.cols, self.cc, self.thresh = list(cols), count_col, thresh
        nt = len(self.cols)
        self.run = np.zeros((3 + nt, n))
        self.win = np.zeros((5 + 2 * nt, n))

    def step(self, reward, done, info):
        nt = len(self.cols)
        ret = self.run[0] + reward.astype(np.float64)
        length = self.run[1] + 1.0
        cnt = self.run[2].copy()
        if self.cc >= 0:
            with np.errstate(invalid="ignore"):
                cnt = cnt + np.where(info[:, self.cc].astype(np.float64) >= self.thresh, 1.0, 0.0)
        term = np.array([self.run[3 + j] + info[:, c].astype(np.float64) for j, c in enumerate(self.cols)]).reshape(nt, len(reward))
        ok = np.isfinite(ret) & np.all(np.isfinite(term), axis=0)
        d = done.astype(bool)
        f, bad = d & ok, d & ~ok
        w = self.win
        w[0, f] += 1.0
        w[2, f] += ret[f]
        w[3, f] += length[f]
        if self.cc >= 0:
            w[4, f] += cnt[f] / length[f]
        for j in range(nt):
            w[5 + j, f] += term[j, f]
            w[5 + nt + j, f] += term[j, f] / length[f]
        w[1, bad] += 1.0
        keep = ~d
        self.run[0] = np.where(keep, ret, 0.0)
        self.run[1] = np.where(keep, length, 0.0)
        self.run[2] = np.where(keep, cnt, 0.0)
        for j in range(nt):
            self.run[3 + j] = np.where(keep, term[j], 0.0)


def _inputs(rng, n, steps, dtype, poison=True):
    """reward [steps,n], done [steps,n] (random, plus done on the first step and on consecutive steps), info [steps,n,56]; NaN and ±inf in
    rewards and columns when poison."""
    reward = rng.normal(size=(steps, n)).astype(dtype)
    info = rng.normal(0.3, 0.5, size=(steps, n, 56)).astype(dtype)
    done = (rng.random((steps, n)) < 0.15).astype(np.uint8)
    done[0, : n // 5] = 1                      # done on the first step
    done[3:6, n // 5: n // 5 + 9] = 1          # done on consecutive steps
    done[-1, :] = 1
    if poison:
        for bad in (np.nan, np.inf, -np.inf):
            reward[rng.integers(0, steps, 6), rng.integers(0, n, 6)] = bad
            info[rng.integers(0, steps, 6), rng.integers(0, n, 6), rng.integers(0, 12, 6)] = bad
    return reward, done, info


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("terms,count", [((), None), (("torso", "feet", "up", "tau", "badfoot", "footcontact"), "velx"), (TERMS16, "velx"),
                                         (TERMS16, None)], ids=["none", "eval_terms", "sixteen", "sixteen_nocount"])
def test_kernel_matches_numpy_bit_for_bit(prec, terms, count):
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import INFO
    from paddlerobotics_b200.es import TrainEpisodeStats
    dt = np.float32 if prec == "f32" else np.float64
    tdt = torch.float32 if prec == "f32" else torch.float64
    n, steps = 1000, 40                         # 1000: the last block of 256 is partial
    rng = np.random.default_rng(11)
    reward, done, info = _inputs(rng, n, steps, dt)
    st = TrainEpisodeStats(_lib.load(), n, torch.device("cuda"), terms, count_col=count)
    ref = RefStats(n, [INFO[k] for k in terms], -1 if count is None else INFO[count])
    for k in range(steps):
        r, d, i = (torch.as_tensor(x, device="cuda") for x in (reward[k], done[k], info[k]))
        assert r.dtype == tdt
        st.step(r, d, i, _stream())
        ref.step(reward[k], done[k], info[k])
        if k in (0, 5, steps - 1):
            np.testing.assert_array_equal(st.run.cpu().numpy(), ref.run)
            np.testing.assert_array_equal(st.win.cpu().numpy(), ref.win)
    w = ref.win
    assert w[1].sum() > 0 and w[0].sum() > 0 and np.isfinite(w).all()      # the poisoned episodes were only counted
    got = st.take()
    assert got["episodes"] == int(w[0].sum()) and got["nonfinite_episodes"] == int(w[1].sum())
    assert got["return"] == pytest.approx(w[2].sum() / w[0].sum(), rel=1e-12) and got["length"] == pytest.approx(w[3].sum() / w[0].sum(), rel=1e-12)
    assert (got["success_rate"] is None) == (count is None)
    assert float(st.win.abs().sum()) == 0.0
    st.restart()
    assert float(st.run.abs().sum()) == 0.0


def test_graph_replay_equals_eager_calls():
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200.es import TrainEpisodeStats
    from paddlerobotics_b200.train import EVAL_TERMS
    n, steps = 777, 12
    reward, done, info = _inputs(np.random.default_rng(5), n, steps, np.float32)
    eager = TrainEpisodeStats(_lib.load(), n, torch.device("cuda"), EVAL_TERMS)
    graphed = TrainEpisodeStats(_lib.load(), n, torch.device("cuda"), EVAL_TERMS)
    r_in, d_in, i_in = (torch.zeros_like(torch.as_tensor(x[0], device="cuda")) for x in (reward, done, info))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        graphed.step(r_in, d_in, i_in, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.current_stream().wait_stream(s)
    graphed.run.zero_(); graphed.win.zero_()
    for k in range(steps):
        r, d, i = (torch.as_tensor(x[k], device="cuda") for x in (reward, done, info))
        eager.step(r, d, i, _stream())
        r_in.copy_(r); d_in.copy_(d); i_in.copy_(i)
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.run, graphed.run) and torch.equal(eager.win, graphed.win)


def test_invalid_arguments_return_minus_one_and_write_nothing():
    import torch
    from paddlerobotics_b200 import _lib
    lib = _lib.load()
    n = 300
    rew, info = torch.randn(n, device="cuda"), torch.randn(n, 56, device="cuda")
    done = torch.ones(n, dtype=torch.uint8, device="cuda")
    run = torch.full((5, n), 7.0, dtype=torch.float64, device="cuda")
    win = torch.full((9, n), 3.0, dtype=torch.float64, device="cuda")
    cols = (C.c_int32 * 16)(1, 2)
    ok = dict(reward=rew.data_ptr(), done=done.data_ptr(), info=info.data_ptr(), info_dim=56, cols=cols, ncols=2, count_col=0, thresh=0.3,
              run=run.data_ptr(), win=win.data_ptr(), n=n, elem_size=4)
    call = lambda a: lib.b2q_train_episode_stats(a["reward"], a["done"], a["info"], a["info_dim"], a["cols"], a["ncols"], a["count_col"], a["thresh"],
                                                 a["run"], a["win"], a["n"], a["elem_size"], _stream())
    bad_cols = (C.c_int32 * 16)(1, 56)
    neg_cols = (C.c_int32 * 16)(-1, 2)
    for change in (dict(reward=None), dict(done=None), dict(run=None), dict(win=None), dict(info=None), dict(cols=None), dict(ncols=-1), dict(ncols=17),
                   dict(cols=bad_cols), dict(cols=neg_cols), dict(count_col=56), dict(count_col=-2), dict(elem_size=2), dict(elem_size=0), dict(n=0),
                   dict(info_dim=0)):
        assert call({**ok, **change}) == -1, change
    torch.cuda.synchronize()
    assert bool((run == 7.0).all()) and bool((win == 3.0).all())
    assert call(ok) == 0
    torch.cuda.synchronize()
    assert not bool((win == 3.0).all())


def test_window_sums_match_episodes_cut_on_the_host():
    """256 auto-reset envs on flat ground, e_step 30, 200 steps of random residuals: every reward / done / info row recorded on the host and
    the episodes cut there in NumPy give the kernel's window, bit for bit."""
    import torch
    from paddlerobotics_b200 import _lib, train
    from paddlerobotics_b200._config import INFO
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.es import TrainEpisodeStats
    args = train.parser().parse_args(["--task_mode", "ground", "--num_envs", "256", "--e_step", "30"])
    env = VecQuadrupedalEnv(256, auto_reset=True, max_episode_steps=30, **train.train_env_config(args))
    w, b = train.initial_etg(args)[1:]
    env.reset(w, b)
    st = TrainEpisodeStats(_lib.load(), 256, env.device, train.EVAL_TERMS)
    g = torch.Generator(device="cuda").manual_seed(3)
    rows = []
    for _ in range(200):
        _, rew, done, info = env.step((torch.rand(256, 12, device="cuda", generator=g) * 2 - 1) * 0.3)
        st.step(rew, done, info, env._stream())
        rows.append((rew.cpu().numpy().copy(), done.cpu().numpy().copy(), info.cpu().numpy().copy()))
    win = st.win.cpu().numpy()
    cols = [INFO[k] for k in train.EVAL_TERMS]
    want = np.zeros_like(win)
    nt = len(cols)
    for e in range(256):                        # per env: cut the recorded stream at every done
        ret = length = cnt = 0.0
        term = [0.0] * nt
        for rew, done, info in rows:
            ret = ret + float(rew[e]); length = length + 1.0
            cnt = cnt + (1.0 if float(info[e, INFO["velx"]]) >= 0.3 else 0.0)
            term = [term[j] + float(info[e, c]) for j, c in enumerate(cols)]
            if done[e]:
                if np.isfinite(ret) and all(np.isfinite(term)):
                    want[0, e] += 1; want[2, e] += ret; want[3, e] += length; want[4, e] += cnt / length
                    for j in range(nt):
                        want[5 + j, e] += term[j]; want[5 + nt + j, e] += term[j] / length
                else:
                    want[1, e] += 1
                ret = length = cnt = 0.0
                term = [0.0] * nt
    np.testing.assert_array_equal(win, want)
    assert want[0].sum() >= 256 * 6 and (want[3] / np.maximum(want[0], 1)).max() <= 30
    env.close()


class _Recorder:
    """Subclasses that record the training env, the replay memory and the learner train.main builds."""

    def __init__(self, monkeypatch, train):
        self.envs, self.rpms, self.learners = [], [], []
        rec = self

        class Env(train.VecQuadrupedalEnv):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                rec.envs.append(self)

        class Rpm(train.ReplayMemory):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                rec.rpms.append(self)

        class Learner(train.SACLearner):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                rec.learners.append(self)
        monkeypatch.setattr(train, "VecQuadrupedalEnv", Env)
        monkeypatch.setattr(train, "ReplayMemory", Rpm)
        monkeypatch.setattr(train, "SACLearner", Learner)


def test_train_records_and_the_evaluation_block(monkeypatch):
    import torch
    from paddlerobotics_b200 import es, train
    rec = _Recorder(monkeypatch, train)
    sums = []
    real_take = es.TrainEpisodeStats.take

    def take(self):
        sums.append(self.win.sum(1).tolist())
        return real_take(self)
    monkeypatch.setattr(es.TrainEpisodeStats, "take", take)
    checks = []
    real_eval = train.run_evaluate_episodes

    def state():
        torch.cuda.synchronize()
        env = [e for e in rec.envs if e.cfg.auto_reset][0]
        rpm, learner = rec.rpms[0], rec.learners[0]
        return (env.get_state().clone(), rpm.cursor.clone(), (rpm._curr_pos, rpm._curr_size, rpm._samples), learner.steps,
                torch.cuda.get_rng_state().clone(), env.obs.clone())

    def wrapped(*a, **k):
        before = state()
        out = real_eval(*a, **k)
        after = state()
        checks.append((before, after))
        return out
    monkeypatch.setattr(train, "run_evaluate_episodes", wrapped)
    n = 256
    log = train.main(["--num_envs", str(n), "--batch", "256", "--warmup_steps", "2048", "--log_every", "5", "--ES", "0", "--task_mode", "ground",
                      "--eval_every_steps", str(10 * n), "--max_steps", str(40 * n), "--train_eval_envs", "2", "--e_step", "40"])
    train_recs = [r for r in log if "iters" in r]
    evals = [r for r in log if "eval_env_steps" in r]
    assert [r["eval_env_steps"] for r in evals] == [10 * n, 20 * n, 30 * n, 40 * n]
    keys = {"train_episodes", "train_nonfinite_episodes", "train_episode_step", "train_success_rate"} | \
        {"train_%s_%s" % (p, k) for p in ("episode", "mean") for k in train.EVAL_TERMS}
    assert all(keys <= set(r) for r in train_recs)
    assert len(sums) == len(train_recs) == 8
    for r, s in zip(train_recs, sums):
        if s[0] > 0:
            assert r["episode_return"] == s[2] / s[0] and r["train_episodes"] == int(s[0]) and r["train_episode_step"] == s[3] / s[0]
        else:
            assert r["episode_return"] is None and r["train_episode_step"] is None
    assert sum(r["train_episodes"] or 0 for r in train_recs) > 0
    for r in evals:
        assert {"eval_episode_reward", "eval_episode_step", "eval_success_rate", "e_step"} <= set(r) and r["e_step"] == 40
        assert {"eval_episode_" + k for k in train.EVAL_TERMS} <= set(r) and np.isfinite(r["eval_episode_reward"])
    assert len(checks) == 4
    for before, after in checks:
        assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1]) and before[2] == after[2] and before[3] == after[3]
        assert torch.equal(before[4], after[4]) and torch.equal(before[5], after[5])


def test_e_step_growth_recaptures_the_iteration_graph():
    """--graph_iter 1 with --act_bound 0 on flat ground: the open-loop gait of --footheight 0.03 --steplen 0.02 walks, so every episode runs to
    the limit in force.  After every growth the window's mean episode length is the new limit: the recaptured graph uses it."""
    from paddlerobotics_b200 import train
    n, every, log_every, e0, g = 256, 100, 10, 100, 50
    log = train.main(["--num_envs", str(n), "--batch", "256", "--warmup_steps", "2048", "--log_every", str(log_every), "--ES", "0",
                      "--task_mode", "ground", "--act_bound", "0", "--footheight", "0.03", "--steplen", "0.02", "--graph_iter", "1",
                      "--e_step", str(e0), "--e_step_growth", str(g), "--eval_every_steps", str(every * n), "--max_steps", str(700 * n)])
    seen = set()
    for r in log:
        it = r["iters"]
        limit = e0
        for blk in range(every, it - log_every + 1, every):     # blocks run after the log record of their iteration
            limit = train.grow_e_step(limit, g)
        assert r["train_nonfinite_episodes"] in (None, 0), r
        if r["train_episodes"]:
            assert r["train_episode_step"] == limit, (it, r["train_episode_step"], limit)
            seen.add(limit)
    assert len(seen) >= 3 and max(seen) > e0, seen


def test_etg_T_reaches_the_step_kernel():
    """--ETG_T 0.4: the first zero-residual step's info['ETG_act'] is the ETG at T = 0.4 (etg.etg_act_table), not at the default 0.5."""
    import torch
    from paddlerobotics_b200 import train
    from paddlerobotics_b200._config import INFO
    from paddlerobotics_b200.etg import etg_act_table
    args = train.parser().parse_args(["--ETG_T", "0.4", "--ETG_T2", "0.4", "--num_envs", "4", "--ES", "0", "--task_mode", "ground"])
    env, _ = train.make_envs(args, train.train_env_config(args))
    _, w, b = train.initial_etg(args)
    env.reset(w, b)
    info = env.step(torch.zeros(4, 12, device="cuda"))[3][:, INFO["ETG_act"]].double().cpu().numpy()
    at4 = etg_act_table(w, b, 1, T=0.4, T2=0.4, t0=0.026)[0]
    at5 = etg_act_table(w, b, 1, T=0.5, T2=0.5, t0=0.026)[0]
    assert np.abs(info - at4).max() < 2e-6
    assert np.abs(info - at5).max() > 1e-3
    env.close()


def test_sensor_widths_and_torque_mode(tmp_path):
    import torch
    from paddlerobotics_b200 import train
    base = ["--num_envs", "256", "--batch", "256", "--warmup_steps", "1024", "--log_every", "5", "--ES", "0", "--task_mode", "ground"]
    train.main(base + ["--sensor_dis", "0", "--max_steps", str(20 * 256), "--outdir", str(tmp_path), "--suffix", "s", "--eval_every_steps", str(10 * 256)])
    pts = sorted(f for f in os.listdir(tmp_path / "s") if f.endswith(".pt"))
    assert pts
    sd = torch.load(tmp_path / "s" / pts[-1])
    assert sd["actor_model.l1.weight"].shape == (256, 46) and sd["critic_model.l1.weight"].shape == (256, 58)
    rec = train.main(["--eval", "1", "--sensor_dis", "0", "--task_mode", "ground", "--load", str(tmp_path / "s" / pts[-1])])
    assert np.isfinite(rec["mean_return"]) and rec["mean_length"] >= 1
    with pytest.raises(SystemExit):                 # the same checkpoint under the full 49-wide observation
        train.main(["--eval", "1", "--task_mode", "ground", "--load", str(tmp_path / "s" / pts[-1])])
    log = train.main(base + ["--act_mode", "torque", "--max_steps", str(20 * 256)])
    losses = [(r["critic_loss"], r["actor_loss"]) for r in log if r.get("critic_loss") is not None]
    assert len(log) == 4 and losses and np.isfinite(losses).all(), log
