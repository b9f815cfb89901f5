"""Behaviour cloning on the device: the student-observation kernel (b2q_bc_observe), the permutation gather on a device cursor
(b2q_bc_gather_cursor), the counter-RNG BC update (b2q_sac_bc_learn_seeded), the graph-replayed sweep (SACLearner.bc_sweep) and the
bctrain command (the batched ETGRL/BCtrain.py), end to end and on the shipped BC checkpoint."""
import ctypes as C
import os

import numpy as np
import pytest

import nets_ref as R

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_PT = os.path.join(HERE, "golden", "StairStair3_BC1_itr_500383.pt")


def _key(seed, step):
    """b2q_bc_observe's Philox key: word 0 = seed, word 1 = step (include/b2q_rpm.h)."""
    return (seed & 0xFFFFFFFF) | ((step & 0xFFFFFFFF) << 32)


def _expected_student(obs, seed, step):
    """obs[:, 3:] + float32(sigma * z) in float32, z = the NumPy Philox draw of (env row, expert column); also the noise terms."""
    from paddlerobotics_b200.bc import NOISE
    n, d = obs.shape
    out, noise = obs[:, 3:].copy(), np.zeros((n, d - 3), np.float32)
    for lo, hi, sig in NOISE:
        z = R.philox_normal(_key(seed, step), np.arange(n)[:, None], np.arange(lo, hi)[None, :]).astype(np.float32)
        noise[:, lo - 3:hi - 3] = np.float32(sig) * z
    noisy = np.zeros(d - 3, bool)
    for lo, hi, _ in NOISE:
        noisy[lo - 3:hi - 3] = True
    out[:, noisy] = out[:, noisy] + noise[:, noisy]
    return out, noise, noisy


def test_observe_student_rows_noise_and_ring_wrap():
    import torch
    from paddlerobotics_b200.bc import BCReplayMemory
    n, cap, seed, step = 1000, 2500, 3, 7
    g = torch.Generator(device="cuda").manual_seed(1)
    obs = torch.randn(n, 49, device="cuda", generator=g) * 2
    m = BCReplayMemory(cap, 46, 49)
    m._pos, m._size = 2000, 2000                                   # the next 1000 rows wrap: slots 2000..2499, 0..499
    before_obs, before_ref = m.obs.clone(), m.ref_obs.clone()
    stu = m.observe(obs, step, seed=seed)
    torch.cuda.synchronize()
    assert m._pos == 500 and m.size() == cap
    slots = (torch.arange(n, device="cuda") + 2000) % cap
    assert torch.equal(m.ref_obs[slots], obs)                       # expert rows: bit for bit
    assert torch.equal(m.obs[slots], stu)
    untouched = torch.ones(cap, dtype=torch.bool, device="cuda"); untouched[slots] = False
    assert torch.equal(m.obs[untouched], before_obs[untouched]) and torch.equal(m.ref_obs[untouched], before_ref[untouched])
    o = obs.cpu().numpy()
    exp, noise, noisy = _expected_student(o, seed, step)
    s = stu.cpu().numpy()
    assert np.array_equal(s[:, ~noisy], o[:, 3:][:, ~noisy])        # columns outside the four slices: exact copies
    # the device's logf / cosf are within 1 / 2 ulp (CUDA math API), sqrtf is correctly rounded: the noise term may differ from the
    # NumPy float64 draw by a few ulp of itself, the float32 add adds at most 1 ulp of the result
    d = np.abs(s[:, noisy] - exp[:, noisy])
    tol = np.spacing(np.abs(exp[:, noisy])) + 4 * np.spacing(np.abs(noise[:, noisy]))
    print("observe: max |student - numpy| = %.3g, in units of the tolerance %.3g" % (d.max(), (d / tol).max()))
    assert (d <= tol).all()
    assert not np.array_equal(s[:, noisy], o[:, 3:][:, noisy])
    # noise off: the whole student row is the slice; a NULL ring writes the student rows only
    ring = (m.obs.clone(), m.ref_obs.clone(), m._pos, m._size)
    s0 = m.observe(obs, step, noise=False, append=False, seed=seed)
    assert torch.equal(s0, obs[:, 3:])
    s1 = m.observe(obs, step, noise=True, append=False, seed=seed)
    assert torch.equal(s1, stu)                                      # same key, same draw
    assert torch.equal(m.obs, ring[0]) and torch.equal(m.ref_obs, ring[1]) and (m._pos, m._size) == ring[2:]
    # another step or seed: another draw
    assert not torch.equal(m.observe(obs, step + 1, append=False, seed=seed), stu)
    assert not torch.equal(m.observe(obs, step, append=False, seed=seed + 1), stu)


def test_observe_noise_statistics_per_slice():
    import torch
    from paddlerobotics_b200.bc import NOISE, BCReplayMemory
    n = 40000
    m = BCReplayMemory(1, 46, 49)
    s = m.observe(torch.zeros(n, 49, device="cuda"), 11, append=False, seed=5).double().cpu().numpy()
    for lo, hi, sig in NOISE:
        x = s[:, lo - 3:hi - 3].reshape(-1) / np.float32(sig)
        k = x.size
        assert k >= 1e5
        assert abs(x.mean()) < 5 / np.sqrt(k), (lo, x.mean())
        assert abs(x.std() - 1) < 5 * np.sqrt(0.5 / k), (lo, x.std())
    assert not s[:, :4].any() and not s[:, 34:].any()


def test_gather_cursor_windows_and_graph_replay():
    import torch
    from paddlerobotics_b200.bc import BCReplayMemory
    cap, B, G = 3001, 128, 3
    m = BCReplayMemory(cap, 46, 49)
    g = torch.Generator(device="cuda").manual_seed(4)
    m.obs.copy_(torch.randn(cap, 46, device="cuda", generator=g)); m.ref_obs.copy_(torch.randn(cap, 49, device="cuda", generator=g))
    perm = torch.randperm(cap, device="cuda", generator=g)
    cur = torch.zeros(1, dtype=torch.int64, device="cuda")
    o, r = torch.zeros(B, 46, device="cuda"), torch.zeros(B, 49, device="cuda")
    m.gather_cursor(perm, cur, o, r)
    assert torch.equal(o, m.obs[perm[:B]]) and torch.equal(r, m.ref_obs[perm[:B]]) and int(cur) == B
    # G gathers captured once; two replays cover the next 2 G windows
    outs = [(torch.zeros(B, 46, device="cuda"), torch.zeros(B, 49, device="cuda")) for _ in range(G)]
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        for oo, rr in outs:
            m.gather_cursor(perm, cur, oo, rr)
    assert int(cur) == B                                             # capturing runs nothing
    for rep in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for k, (oo, rr) in enumerate(outs):
            idx = perm[(1 + rep * G + k) * B:(2 + rep * G + k) * B]
            assert torch.equal(oo, m.obs[idx]) and torch.equal(rr, m.ref_obs[idx]), (rep, k)
    assert int(cur) == (1 + 2 * G) * B
    # rows past the end of perm are not written
    cur.fill_(cap - 50)
    o.fill_(7.0); r.fill_(7.0)
    m.gather_cursor(perm, cur, o, r)
    assert torch.equal(o[:50], m.obs[perm[cap - 50:]]) and bool((o[50:] == 7).all()) and bool((r[50:] == 7).all())
    # iter_pass: range(0, size - batch, batch) windows of one permutation
    got = [x[1].clone() for x in m.iter_pass(B, size=1000, generator=torch.Generator(device="cuda").manual_seed(9))]
    p2 = torch.randperm(1000, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    assert len(got) == len(range(0, 1000 - B, B)) == 7
    for k, x in enumerate(got):
        assert torch.equal(x, m.ref_obs[p2[k * B:(k + 1) * B]])


def _seeded(L, obs, ref, expert, eps, seed):
    rc = L.lib.b2q_sac_bc_learn_seeded(L.h, obs.data_ptr(), ref.data_ptr(), ref.shape[1], expert.actor.h, expert.critic.h,
                                       None if eps is None else eps.data_ptr(), C.c_uint64(seed), None, L._stream())
    assert rc == 0, rc


def _rel(x, y):
    return float((x - y).norm() / max(float(y.norm()), 1e-30))


TOL_RNG = 8e-4     # the counter-RNG draw vs the NumPy Philox draw, up to the order of the split-K atomics (test_gpu_sac's bound)


def test_seeded_bc_update_draws_the_numpy_philox_noise():
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    B, A, seed = 256, 12, 1234
    expert = MujocoAgent(49, A, seed=21)
    Ls = [SACLearner(MujocoAgent(46, A, seed=22), B) for _ in range(2)]
    g = torch.Generator(device="cuda").manual_seed(3)
    worst = 0.0
    for t in range(3):
        ref = torch.randn(B, 49, device="cuda", generator=g)
        obs = ref[:, 3:].contiguous()
        _seeded(Ls[0], obs, ref, expert, None, seed)
        eps = torch.as_tensor(R.philox_eps(R.effective_seed(seed, t), B, A), device="cuda")     # ctr = completed steps = t
        assert Ls[1].lib.b2q_sac_bc_learn(Ls[1].h, obs.data_ptr(), ref.data_ptr(), 49, expert.actor.h, expert.critic.h, eps.data_ptr(), None, Ls[1]._stream()) == 0
        l0, l1 = Ls[0].losses.clone(), Ls[1].losses.clone()
        torch.cuda.synchronize()
        assert _rel(l0.double(), l1.double()) < 1e-4, (l0, l1)
        for x, y in zip(Ls[0].grads(), Ls[1].grads()):
            worst = max(worst, _rel(x.double(), y.double()))
    print("seeded BC update vs explicit numpy eps: worst gradient rel L2 %.3g" % worst)
    assert worst < TOL_RNG
    # the explicit-eps entry point is the seeded one with eps given, and still refuses a NULL eps
    L = Ls[1]
    assert L.lib.b2q_sac_bc_learn(L.h, obs.data_ptr(), ref.data_ptr(), 49, expert.actor.h, expert.critic.h, None, None, L._stream()) == -1


def test_bc_learn_with_eps_is_unchanged_by_the_seeded_entry_point():
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
    B = 256
    expert = MujocoAgent(49, 12, seed=5)
    res = []
    for path in ("bc_learn", "seeded"):
        st = MujocoAgent(46, 12, seed=6)
        L = SACLearner(st, B)
        g = torch.Generator(device="cuda").manual_seed(8)
        for _ in range(3):
            ref, eps = torch.randn(B, 49, device="cuda", generator=g), torch.randn(B, 12, device="cuda", generator=g)
            obs = ref[:, 3:].contiguous()
            if path == "bc_learn":
                L.bc_learn(obs, ref, expert, eps=eps, pull=False)
            else:
                _seeded(L, obs, ref, expert, eps, 99)
        L.pull()
        res.append(flatten_params(st.params))
    for x, y in zip(*res):
        assert float((x - y).abs().max()) < 2e-5          # split-K f32 atomics reorder sums run to run; otherwise identical


def test_bc_sweep_graph_replay_equals_eager_seeded_updates():
    """K = 2 G + 3 updates: two graph replays and an eager remainder of 3, against K eager seeded updates on the same batches.  Both run
    the same kernels with the same counter-RNG keys; what differs is the order of the f32 atomics in the split-K weight gradients and
    bias sums, so parameters agree to a few 1e-5 (test_sac_learn_cuda_graph_replay_equals_eager's bound) and losses to 1e-4 relative."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
    from paddlerobotics_b200.bc import BCReplayMemory
    B, G, seed = 256, 4, 17
    K = 2 * G + 3
    expert = MujocoAgent(49, 12, seed=31)
    m = BCReplayMemory(K * B + 100, 46, 49)
    g = torch.Generator(device="cuda").manual_seed(2)
    ref = torch.randn(m.max_size, 49, device="cuda", generator=g)
    m.ref_obs.copy_(ref); m.obs.copy_(ref[:, 3:])
    perm = torch.randperm(m.max_size, device="cuda", generator=g)
    st_g, st_e = MujocoAgent(46, 12, seed=32), MujocoAgent(46, 12, seed=32)
    Lg, Le = SACLearner(st_g, B), SACLearner(st_e, B)
    mean = Lg.bc_sweep(m, expert, perm, K, seed=seed, graph_steps=G)
    acc = torch.zeros(2, device="cuda")
    for k in range(K):
        idx = perm[k * B:(k + 1) * B]
        _seeded(Le, m.obs[idx].contiguous(), m.ref_obs[idx].contiguous(), expert, None, seed)
        acc += Le.losses
    Le.pull()
    torch.cuda.synchronize()
    assert _rel(mean.double(), (acc / K).double()) < 1e-4, (mean, acc / K)
    worst = max(float((x - y).abs().max()) for x, y in zip(flatten_params(st_g.params), flatten_params(st_e.params)))
    print("bc_sweep vs eager: max |param diff| %.3g after %d updates" % (worst, K))
    assert worst < 5e-5
    # a second sweep reuses the captured graph (same pointers) and continues from the updated parameters
    assert len(Lg._bc_graphs) == 1
    Lg.bc_sweep(m, expert, perm, G, seed=seed, graph_steps=G)
    assert len(Lg._bc_graphs) == 1


def test_set_max_episode_steps_changes_the_auto_reset_length():
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.03, Steplength=0.02)
    env = VecQuadrupedalEnv(8, auto_reset=True, max_episode_steps=50)
    env.reset(w, b)
    a = torch.zeros(8, 12, device="cuda")
    env.set_max_episode_steps(3)
    dones = [bool(env.step(a)[2].all()) for _ in range(6)]
    assert dones == [False, False, True, False, False, True]
    env.close()


def _expert_files(tmp_path):
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    MujocoAgent(49, 12, seed=1).save(str(tmp_path / "expert.pt"))
    np.savez(tmp_path / "expert.npz", w=w, b=b)
    return str(tmp_path / "expert.pt"), str(tmp_path / "expert.npz")


def test_bctrain_end_to_end(tmp_path):
    import torch
    from paddlerobotics_b200 import bctrain
    pt, npz = _expert_files(tmp_path)
    n, steps = 512, 512 * 24
    log = bctrain.main(["--ref_agent", pt, "--ETG_path", npz, "--num_envs", str(n), "--max_steps", str(steps), "--memory", "100000",
                        "--eval_every_steps", "4096", "--eval_envs", "8", "--outdir", str(tmp_path), "--suffix", "t", "--graph_steps", "8"])
    train = [r for r in log if "actor_loss" in r]
    evals = [r for r in log if "ref_ratio" in r]
    a = np.array([r["actor_loss"] for r in train])
    print("BC actor loss per training step:", np.round(a, 3))
    assert len(a) >= 10 and np.isfinite(a).all()
    assert a[-2:].mean() < a[:2].mean() - 0.05, (a[:2], a[-2:])        # test_bc_loop_clones_expert's margin
    expected = sum(len(o) for it in range(steps // n) for _, _, o, _ in bctrain.sweep_schedule(it * n, n, 1024, 10, 1024, 100000, 200, 8))
    assert expected == 10 * sum(k - 1 for k in range(1, steps // 1024 + 1))
    assert sum(r["updates"] for r in train) == train[-1]["total_updates"] == expected
    assert len(evals) == 4 and all(r["ref_ratio"] is not None and np.isfinite(r["ref_ratio"]) for r in evals)
    assert train[-1]["e_step"] == 550                                       # 400 + 50 per evaluation before the last training step
    pts = sorted(f for f in os.listdir(tmp_path / "t") if f.startswith("itr_") and f.endswith(".pt"))
    assert pts
    sd, gold = torch.load(tmp_path / "t" / pts[-1], map_location="cpu"), torch.load(GOLDEN_PT, map_location="cpu")
    assert set(sd) == set(gold) and all(tuple(sd[k].shape) == tuple(gold[k].shape) for k in gold)


def test_bctrain_eval_of_the_shipped_student(tmp_path):
    from paddlerobotics_b200 import bctrain
    gait = os.path.join(os.path.dirname(HERE), "paddlerobotics_b200", "data", "etg_shipped_gait.npz")
    rec = bctrain.main(["--eval", "1", "--load", GOLDEN_PT, "--ETG_path", gait, "--render_dir", str(tmp_path), "--render_width", "64",
                        "--render_height", "48", "--eval_envs", "4"])
    assert np.isfinite(rec["mean_return"]) and 1 <= rec["mean_length"] <= 601 and all(np.isfinite(v) for v in rec["terms"].values())
    frames = [f for f in os.listdir(tmp_path) if f.startswith("img") and f.endswith(".png")]
    assert "img1.png" in frames and len(frames) >= 1
