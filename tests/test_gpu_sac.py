"""K5/K6: SAC.learn on the device vs a plain PyTorch fp32 restatement of ETGRL/alg/sac.py:77-118 (same minibatch, same
N(0,1) draws for both rsample() calls).  Forward/backward GEMMs run in bf16 on wgmma tensor cores with f32 accumulation, so the
tolerance is the bf16 one: losses within 2 %, gradient buckets within 5 % relative L2 error and cosine >= 0.995."""
import os

import numpy as np
import pytest

import nets_ref as R
from sac_torch import torch_sac_losses as _torch_sac_step

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [256, 1024])
def test_sac_gradients_and_losses_vs_torch(B):
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
    torch.manual_seed(B)
    ag = MujocoAgent(49, 12, seed=5)
    gamma, alpha = 0.99, 0.2
    L = SACLearner(ag, B, gamma=gamma, tau=0.005, alpha=alpha, actor_lr=3e-4, critic_lr=3e-4)
    dev = ag.device
    obs, nobs = torch.randn(B, 49, device=dev), torch.randn(B, 49, device=dev)
    act = torch.rand(B, 12, device=dev) * 2 - 1
    rew, term = torch.randn(B, device=dev), (torch.rand(B, device=dev) > 0.1).float()
    e1, e2 = torch.randn(B, 12, device=dev), torch.randn(B, 12, device=dev)
    p = {k: v.clone().requires_grad_(True) for k, v in ag.params.items()}
    tgt = {k: v.clone() for k, v in ag.params.items()}
    cl, al = _torch_sac_step(p, tgt, obs, act, rew, nobs, term, e1, e2, gamma, alpha)
    gc = torch.autograd.grad(cl, [p[k] for k in p if k.startswith("critic")], retain_graph=True)
    ga = torch.autograd.grad(al, [p[k] for k in p if k.startswith("actor")])
    gp = {k: g for k, g in zip([k for k in p if k.startswith("critic")], gc)}
    gp.update({k: g for k, g in zip([k for k in p if k.startswith("actor")], ga)})
    ref_a, ref_c = flatten_params(gp)
    # device: gradient phases only (0 and 2), no optimiser step in between, so both are taken at the same parameters
    lib, h, st = L.lib, L.h, L._stream()
    args = (obs.data_ptr(), act.data_ptr(), rew.data_ptr(), nobs.data_ptr(), term.data_ptr(), e1.data_ptr(), e2.data_ptr(), 1)
    assert lib.b2q_sac_phase(h, 0, *args, st) == 0
    assert lib.b2q_sac_phase(h, 2, *args, st) == 0
    ga_d, gc_d = L.grads()
    losses = torch.as_tensor(__import__("paddlerobotics_b200.agent", fromlist=["_CudaBuf"])._CudaBuf(lib.b2q_sac_loss_ptr(h), 2), device=dev).clone()
    torch.cuda.synchronize()
    cl, al = cl.detach(), al.detach()
    assert abs(float(losses[0]) - float(cl)) < 0.02 * abs(float(cl)) + 1e-3, (float(losses[0]), float(cl))
    assert abs(float(losses[1]) - float(al)) < 0.02 * abs(float(al)) + 2e-2, (float(losses[1]), float(al))
    for name, d, r in (("critic", gc_d, ref_c), ("actor", ga_d, ref_a)):
        rel = float((d - r).norm() / r.norm())
        cos = float(torch.dot(d, r) / (d.norm() * r.norm()))
        print(name, "grad rel L2 err %.4f cos %.5f" % (rel, cos))
        assert rel < 0.05 and cos > 0.995, (name, rel, cos)


def test_sac_learn_three_steps_tracks_torch_adam():
    """Full learn() (critic Adam -> actor grads at the UPDATED critic -> actor Adam -> Polyak), 3 steps, vs torch.optim.Adam."""
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
    B, gamma, alpha, tau = 256, 0.99, 0.2, 0.005
    torch.manual_seed(0)
    ag = MujocoAgent(49, 12, seed=9)
    L = SACLearner(ag, B, gamma=gamma, tau=tau, alpha=alpha, actor_lr=3e-4, critic_lr=3e-4)
    dev = ag.device
    p = {k: v.clone().requires_grad_(True) for k, v in ag.params.items()}
    tgt = {k: v.clone() for k, v in ag.params.items()}
    opt_a = torch.optim.Adam([p[k] for k in p if k.startswith("actor")], lr=3e-4)
    opt_c = torch.optim.Adam([p[k] for k in p if k.startswith("critic")], lr=3e-4)
    a0, c0 = flatten_params(ag.params)
    for step in range(3):
        obs, nobs = torch.randn(B, 49, device=dev), torch.randn(B, 49, device=dev)
        act = torch.rand(B, 12, device=dev) * 2 - 1
        rew, term = torch.randn(B, device=dev), (torch.rand(B, device=dev) > 0.1).float()
        e1, e2 = torch.randn(B, 12, device=dev), torch.randn(B, 12, device=dev)
        cl, _ = _torch_sac_step(p, tgt, obs, act, rew, nobs, term, e1, e2, gamma, alpha)
        opt_c.zero_grad(); cl.backward(); opt_c.step()
        _, al = _torch_sac_step(p, tgt, obs, act, rew, nobs, term, e1, e2, gamma, alpha)
        opt_a.zero_grad(); al.backward(); opt_a.step()
        with torch.no_grad():
            for k in tgt:
                tgt[k].copy_(tau * p[k] + (1 - tau) * tgt[k])
        losses = L.learn(obs, act, rew, nobs, term, eps_next=e1, eps_cur=e2)
        assert abs(float(losses[0]) - float(cl)) < 0.03 * abs(float(cl)) + 1e-3
        assert abs(float(losses[1]) - float(al)) < 0.03 * abs(float(al)) + 3e-2
    a1, c1 = flatten_params(ag.params)            # pulled back from the learner
    ra, rc = flatten_params({k: v.detach() for k, v in p.items()})
    # the 3-step parameter displacement agrees in direction and size (Adam's sign-like update amplifies tiny gradient noise
    # on near-zero gradients, so compare displacements, not parameters)
    for name, d, r, z in (("actor", a1, ra, a0), ("critic", c1, rc, c0)):
        dd, rr = d - z, r - z
        cos = float(torch.dot(dd, rr) / (dd.norm() * rr.norm()))
        print(name, "3-step displacement cos %.4f, |d| %.4g vs %.4g" % (cos, float(dd.norm()), float(rr.norm())))
        assert cos > 0.9 and 0.8 < float(dd.norm() / rr.norm()) < 1.25
    # agent.learn surface (numpy in, floats out)
    c_l, a_l = ag.learn(obs.cpu().numpy(), act.cpu().numpy(), rew.cpu().numpy(), nobs.cpu().numpy(), term.cpu().numpy())
    assert isinstance(c_l, float) and isinstance(a_l, float) and np.isfinite(c_l) and np.isfinite(a_l)


def test_optimiser_kernels_repack_forward_images_and_backward_copies():
    """The Adam / Polyak kernels write the updated parameters straight into the tensor-core operand images and the bf16 backward copies.
    After three learns they must equal what the stand-alone pack kernels produce from the same f32 parameters: forward outputs bit-equal,
    gradients equal up to the order of the split-K atomics (tau = 1 so that a fresh learner's targets equal the trained one's)."""
    import copy
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    B = 256
    g = torch.Generator(device="cuda"); g.manual_seed(21)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    ag = MujocoAgent(49, 12, seed=13)
    L = SACLearner(ag, B, tau=1.0)
    for _ in range(3):
        L.learn(r(B, 49), torch.rand(B, 12, device="cuda", generator=g) * 2 - 1, r(B), r(B, 49), torch.ones(B, device="cuda"), eps_next=r(B, 12), eps_cur=r(B, 12))
    obs, act = r(B, 49), torch.rand(B, 12, device="cuda", generator=g) * 2 - 1
    # forward images: the learner's nets (written by k_adam_pack) vs the agent's own nets (pack kernel on the pulled parameters)
    from paddlerobotics_b200.agent import PREDICT, RAW
    assert torch.equal(L.actor.forward(obs, mode=PREDICT)[0][0], ag.predict_batch(obs))
    q_l = L.critic.forward(obs, in2=act, mode=RAW)[0]
    q_a = ag.q_values(obs, act)
    assert torch.equal(q_l[0, :, 0], q_a[0]) and torch.equal(q_l[1, :, 0], q_a[1])
    # backward copies and target images: gradient phases of the trained learner vs a fresh learner built from the pulled parameters
    ag2 = MujocoAgent(49, 12, seed=99)
    ag2.load_state_dict(copy.deepcopy(ag.state_dict()))
    L2 = SACLearner(ag2, B, tau=1.0)
    rew, nobs, term, e1, e2 = r(B), r(B, 49), torch.ones(B, device="cuda"), r(B, 12), r(B, 12)
    out = []
    for lr in (L, L2):
        args = (obs.data_ptr(), act.data_ptr(), rew.data_ptr(), nobs.data_ptr(), term.data_ptr(), e1.data_ptr(), e2.data_ptr(), 1)
        assert lr.lib.b2q_sac_phase(lr.h, 0, *args, lr._stream()) == 0
        assert lr.lib.b2q_sac_phase(lr.h, 2, *args, lr._stream()) == 0
        out.append([x.clone() for x in lr.grads()])
    torch.cuda.synchronize()
    for x, y in zip(out[0], out[1]):
        assert float((x - y).abs().max()) <= 1e-5 * float(y.abs().max()) + 1e-9, float((x - y).abs().max())


def rng_metrics(seed):
    """eps = None: both rsample() draws come from the counter RNG inside the kernels.  A learner fed the numpy Philox draws of the keys the
    code uses as explicit eps must produce the same gradients, up to the order of the split-K atomics: eager learn() (keys 2 s + 1 for the next
    observation and 2 s for the current one, s = learner.steps) and CUDA-graph replays 1-3 (host seed 0), both advanced by
    ctr * 0x9E3779B97F4A7C15 with ctr the device step counter.  Returns the worst relative L2 gradient difference of each path."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    B, A = 256, 12
    worst = {}
    for path in ("eager", "graph"):
        Ls = [SACLearner(MujocoAgent(49, A, seed=17 + seed), B) for _ in range(2)]
        w = 0.0
        for t in range(1, 4):
            g = torch.Generator(device="cuda"); g.manual_seed(31 + 10 * seed + t)
            r = lambda *s: torch.randn(*s, device="cuda", generator=g)
            obs, nobs, act, rew, term = r(B, 49), r(B, 49), torch.rand(B, A, device="cuda", generator=g) * 2 - 1, r(B), torch.ones(B, device="cuda")
            if path == "eager":
                Ls[0].learn(obs, act, rew, nobs, term, pull=False)
                s, ctr = Ls[0].steps, t - 1
            else:
                Ls[0].learn(obs, act, rew, nobs, term, pull=False, graph=True)
                s, ctr = 0, t - 1
            e_next = torch.as_tensor(R.philox_eps(R.effective_seed(2 * s + 1, ctr), B, A), device="cuda")
            e_cur = torch.as_tensor(R.philox_eps(R.effective_seed(2 * s, ctr), B, A), device="cuda")
            Ls[1].learn(obs, act, rew, nobs, term, eps_next=e_next, eps_cur=e_cur, pull=False)
            torch.cuda.synchronize()
            for x, y in zip(Ls[0].grads(), Ls[1].grads()):
                w = max(w, _rel(x.double(), y.double()))
        worst[path] = w
        for L in Ls:
            L.close()
    return worst


TOL_RNG = 8e-4      # measured 1.8e-4 eager, 1.9e-5 graph replays


def test_counter_rng_noise_is_the_same_draw_in_forward_and_backward():
    w = rng_metrics(0)
    assert w["eager"] < TOL_RNG and w["graph"] < TOL_RNG, w


def test_graph_learn_without_eps_draws_fresh_noise_and_takes_static_inputs():
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    from paddlerobotics_b200.replay import ReplayMemory
    B = 256
    ag = MujocoAgent(49, 12, seed=3)
    L = SACLearner(ag, B)
    rpm = ReplayMemory(4096, 49, 12)
    g = torch.Generator(device="cuda"); g.manual_seed(2)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    rpm.append(r(2048, 49), torch.rand(2048, 12, device="cuda", generator=g) * 2 - 1, r(2048), r(2048, 49), torch.ones(2048, device="cuda"))
    batch = rpm.sample_batch(B, seed=1, out=L.static_batch())
    assert all(x.data_ptr() == y.data_ptr() for x, y in zip(batch, L.static_batch()))
    losses = []
    for _ in range(3):   # same inputs, no parameter pull: the actor loss changes through the new noise (and the updated nets)
        losses.append(L.learn(*batch, graph=True, pull=False).clone())
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(x).all()) for x in losses)
    assert float((losses[0] - losses[1]).abs().max()) > 0 and float((losses[1] - losses[2]).abs().max()) > 0
    with pytest.raises(ValueError):
        L.learn(*batch, eps_next=r(B, 12), eps_cur=r(B, 12), graph=True, pull=False)


def test_sac_learn_cuda_graph_replay_equals_eager():
    """learn() replayed from a CUDA graph (device-side Adam step counter) == the eager sequence of launches."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
    B = 256
    torch.manual_seed(1)
    res = []
    for use_graph in (False, True):
        ag = MujocoAgent(49, 12, seed=11)
        L = SACLearner(ag, B)
        g = torch.Generator(device="cuda"); g.manual_seed(5)
        for step in range(4):
            r = lambda *s: torch.randn(*s, device="cuda", generator=g)
            obs, nobs, act, rew, term, e1, e2 = r(B, 49), r(B, 49), torch.rand(B, 12, device="cuda", generator=g) * 2 - 1, r(B), torch.ones(B, device="cuda"), r(B, 12), r(B, 12)
            L.learn(obs, act, rew, nobs, term, eps_next=e1, eps_cur=e2, graph=use_graph)
        res.append(flatten_params(ag.params))
        L.close()
    for x, y in zip(res[0], res[1]):
        d = (x - y).abs().max()
        assert d < 2e-5, float(d)      # split-K f32 atomics reorder sums run to run; otherwise identical


def test_bc_learn_vs_torch():
    """f-3: BC.BClearn (alg/BC.py:53-72) — partial-observation student (obs[3:], BCtrain.py:77-81) cloned from an expert:
    actor NLL step then critic regression onto the expert's twin Q, vs a torch fp32 restatement with the same eps."""
    import torch
    import torch.nn.functional as F
    torch.backends.cuda.matmul.allow_tf32 = False
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, flatten_params
    B = 256
    torch.manual_seed(2)
    expert, student = MujocoAgent(49, 12, seed=21), MujocoAgent(46, 12, seed=22)
    L = SACLearner(student, B, actor_lr=3e-4, critic_lr=3e-4)
    dev = student.device
    ref_obs = torch.randn(B, 49, device=dev)
    obs = ref_obs[:, 3:].contiguous()
    eps = torch.randn(B, 12, device=dev)
    p = {k: v.clone().requires_grad_(True) for k, v in student.params.items()}
    pe = expert.params
    a0, c0 = flatten_params(student.params)

    def actor(pp, o):
        x = F.relu(F.linear(o, pp["actor_model.l1.weight"], pp["actor_model.l1.bias"]))
        x = F.relu(F.linear(x, pp["actor_model.l2.weight"], pp["actor_model.l2.bias"]))
        return F.linear(x, pp["actor_model.mean_linear.weight"], pp["actor_model.mean_linear.bias"]), \
            torch.clamp(F.linear(x, pp["actor_model.std_linear.weight"], pp["actor_model.std_linear.bias"]), -20.0, 2.0)

    def critic(pp, o, a):
        x = torch.cat([o, a], 1); out = []
        for l1, l2, l3 in (("l1", "l2", "l3"), ("l4", "l5", "l6")):
            h = F.relu(F.linear(x, pp["critic_model.%s.weight" % l1], pp["critic_model.%s.bias" % l1]))
            h = F.relu(F.linear(h, pp["critic_model.%s.weight" % l2], pp["critic_model.%s.bias" % l2]))
            out.append(F.linear(h, pp["critic_model.%s.weight" % l3], pp["critic_model.%s.bias" % l3]))
        return out
    opt_a = torch.optim.Adam([p[k] for k in p if k.startswith("actor")], lr=3e-4)
    opt_c = torch.optim.Adam([p[k] for k in p if k.startswith("critic")], lr=3e-4)
    mean, ls = actor(p, obs)
    with torch.no_grad():
        ref_action = torch.tanh(actor(pe, ref_obs)[0])
    actor_loss = -torch.distributions.Normal(mean, ls.exp()).log_prob(ref_action).mean()
    opt_a.zero_grad(); actor_loss.backward(); opt_a.step()
    with torch.no_grad():
        m2, l2 = actor(p, obs)
        a_now = torch.tanh(m2 + l2.exp() * eps)
        rq1, rq2 = critic(pe, ref_obs, a_now)
    q1, q2 = critic(p, obs, a_now)
    critic_loss = F.mse_loss(q1, rq1) + F.mse_loss(q2, rq2)
    opt_c.zero_grad(); critic_loss.backward(); opt_c.step()
    losses = L.bc_learn(obs, ref_obs, expert, eps=eps)
    assert abs(float(losses[1]) - float(actor_loss)) < 0.02 * abs(float(actor_loss)) + 1e-2
    assert abs(float(losses[0]) - float(critic_loss)) < 0.03 * abs(float(critic_loss)) + 1e-3
    a1, c1 = flatten_params(student.params)
    ra, rc = flatten_params({k: v.detach() for k, v in p.items()})
    for name, d, r, z in (("actor", a1, ra, a0), ("critic", c1, rc, c0)):
        dd, rr = d - z, r - z
        cos = float(torch.dot(dd, rr) / (dd.norm() * rr.norm()))
        print(name, "BC displacement cos %.4f |d| %.4g vs %.4g" % (cos, float(dd.norm()), float(rr.norm())))
        assert cos > 0.95 and 0.9 < float(dd.norm() / rr.norm()) < 1.1
    c_l, a_l = student.BClearn(obs, ref_obs, expert)
    assert np.isfinite(c_l) and np.isfinite(a_l)


# ---------------------------------------------------------------------------------------------------------------------------------
# Per-tensor parity with the float64 reference of tests/nets_ref.py.  `mirror` rounds to bf16 where the kernels round, so its distance
# from the device is the kernels' own f32 arithmetic (accumulation order, split-K atomics); `exact` is the true gradient of sac.py.
# Bounds are about 4x the largest value measured on an H100 (80GB HBM3) over seeds 0, 1, 2 of every case; the measured value is beside each.
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CKPT = os.path.join(GOLDEN_DIR, "StairStair3_BC1_itr_500383.pt")
GAMMA, ALPHA, TAU, LR_A, LR_C = 0.99, 0.2, 0.005, 3e-4, 1e-3
#        obs  act  batch  parameters   (B / 64 K-chunks of the weight-gradient GEMMs, split-K splits of 8 chunks at the default B2Q_GEMM_SPLIT_DIV)
SAC_CASES = {"a": (49, 12, 256, "fresh"),     # today's shape, 4 chunks, no split
             "b": (49, 12, 8192, "fresh"),    # the bench batch: 64 row tiles, 128 chunks in 16 splits
             "c": (46, 12, 2176, "ckpt"),     # shipped checkpoint: upper log-std clamp, tanh saturation, |Q| ~ 300; 34 chunks -> 9 + 9 + 9 + 7
             "d": (52, 12, 1664, "fresh"),    # critic in_dim = 64 (no K padding); 26 chunks -> 9 + 9 + 8
             "e": (3, 1, 128, "fresh"),       # A = 1: the runtime-dimension actor head, one tile, no split
             "f": (20, 7, 4096, "clamp")}     # log-std bias -25 on actions 0, 1 and +3 on 2, 3: both clamps; odd A
# relative L2 error per tensor / per loss
TOL_MIRROR = {"a": 6e-4,    # measured 1.5e-4 (critic l4.weight)
              "b": 3e-4,    # measured 6.8e-5 (actor l1.weight)
              "c": 8e-4,    # measured 1.9e-4 (critic l1.weight)
              "d": 8e-3,    # measured 2.0e-3 (critic l4.weight)
              "e": 1e-3,    # measured 2.5e-4 (critic l1.weight)
              "f": 1.1e-3}  # measured 2.6e-4 (critic l1.weight)
TOL_EXACT, COS_EXACT = 0.3, 0.987      # measured 0.079 and cos 0.9969 (critic l4.weight, case e: batch 128)
TOL_LOSS_MIRROR, TOL_LOSS_EXACT = 5e-4, 3e-2     # measured 1.1e-4 (critic loss, case f) and 7.0e-3 (actor loss, case e)


def _rel(d, r):
    return float((d - r).norm() / r.norm().clamp_min(1e-30))


def _cos(d, r):
    return float((d * r).sum() / (d.norm() * r.norm()).clamp_min(1e-30))


def _make_learner(obs_dim, act_dim, B, params, seed, sync="exact"):
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    ag = MujocoAgent(obs_dim, act_dim, seed=100 + seed)
    if params == "ckpt":
        ag.restore(CKPT)
    elif params == "clamp":
        ag.params["actor_model.std_linear.bias"][:2] = -25.0
        ag.params["actor_model.std_linear.bias"][2:4] = 3.0
        ag.sync_weights()
    return ag, SACLearner(ag, B, gamma=GAMMA, tau=TAU, alpha=ALPHA, actor_lr=LR_A, critic_lr=LR_C, sync=sync)


def _sac_batch(obs_dim, act_dim, B, params, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(1000 + seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    if params == "ckpt":      # the golden observations of the shipped policy, tiled, plus N(0, 0.3^2)
        base = torch.tensor(np.load(os.path.join(GOLDEN_DIR, "reference_vectors.npz"))["mlp_obs"], device="cuda")
        obs, nobs = (base.repeat(B // 16 + 1, 1)[:B] + 0.3 * r(B, obs_dim) for _ in range(2))
    else:
        obs, nobs = r(B, obs_dim), r(B, obs_dim)
    return dict(obs=obs.contiguous(), act=torch.rand(B, act_dim, device="cuda", generator=g) * 2 - 1, rew=r(B), nobs=nobs.contiguous(),
                term=(torch.rand(B, device="cuda", generator=g) > 0.1).float(), eps_next=r(B, act_dim), eps_cur=r(B, act_dim))


def _state(L, which=("actor", "critic", "target")):
    """The learner's parameters as state dicts (float32, device): actor + critics, and the target critics."""
    import torch
    from paddlerobotics_b200.agent import unflatten_params
    a, c, t = torch.empty(L.na, device="cuda"), torch.empty(L.nc, device="cuda"), torch.empty(L.nc, device="cuda")
    assert L.lib.b2q_sac_get_params(L.h, a.data_ptr(), c.data_ptr(), t.data_ptr(), L._stream()) == 0
    p, tg = dict(L.agent.params), dict(L.agent.params)
    unflatten_params(p, a, c, L.agent.obs_dim, L.agent.act_dim)
    unflatten_params(tg, a, t, L.agent.obs_dim, L.agent.act_dim)
    return p, {k: v for k, v in tg.items() if k.startswith("critic")}, (a, c, t)


def _dev_grads(L):
    from paddlerobotics_b200.agent import unflatten_params
    a, c = L.grads()
    g = dict(L.agent.params)
    unflatten_params(g, a, c, L.agent.obs_dim, L.agent.act_dim)
    return g, (a, c)


def _phase_args(b, eps=True):
    pe = lambda x: x.data_ptr() if eps else None
    return (b["obs"].data_ptr(), b["act"].data_ptr(), b["rew"].data_ptr(), b["nobs"].data_ptr(), b["term"].data_ptr(), pe(b["eps_next"]), pe(b["eps_cur"]), 1)


def _b64(b):
    return {k: v.double() for k, v in b.items()}


def _compare(dev, mirror, exact, critic_loss):
    """Per-tensor metrics: mirror rel. L2, exact rel. L2 and cosine; asserts exact zeros (where mirror and exact are both 0) on the device.
    The critic heads' bias gradient sum_b 2 (q_b - tq_b) / B can cancel to almost nothing; it is measured against the bound of its summands,
    sum_b |2 (q_b - tq_b) / B| <= 2 sqrt(critic_loss), instead of its own size."""
    out = {}
    for k in exact:
        d = dev[k].double()
        both0 = (mirror[k] == 0) & (exact[k] == 0)
        assert float(d[both0].abs().max()) == 0.0 if bool(both0.any()) else True, (k, "nonzero device gradient where the reference is 0")
        if k in ("critic_model.l3.bias", "critic_model.l6.bias"):
            s = 2 * float(critic_loss) ** 0.5
            out[k] = (float((d - mirror[k]).norm()) / s, float((d - exact[k]).norm()) / s, 1.0)
        else:
            out[k] = (_rel(d, mirror[k]), _rel(d, exact[k]), _cos(d, exact[k]))
    return out


def _phase2_forward(L, obs, eps):
    """The sampled actions and raw log-std of phase 2's actor forward, recomputed with the same kernel and operand images (bit-identical: the
    forward has no atomics).  Call it while the actor still has the parameters phase 2 used."""
    from paddlerobotics_b200.agent import SAMPLE
    out, _, raw = L.actor.forward(obs, mode=SAMPLE, eps=eps, want_raw=True)
    return {"a": out[0], "raw_ls": raw[0, :, L.agent.act_dim:]}


def _phase2_q(L, obs, dev):
    """Adds the twin Q at those actions, from the critics as phase 2 saw them (in learn(): after the critics' optimiser step)."""
    from paddlerobotics_b200.agent import RAW
    q = L.critic.forward(obs, in2=dev["a"], mode=RAW)[0]
    dev["q"] = (q[0, :, 0], q[1, :, 0])
    return dev


def sac_case_metrics(case, seed):
    """Flat phase order (0 then 2, both gradients at the same parameters): per-tensor and loss errors of case `case` with seed `seed`."""
    import torch
    from paddlerobotics_b200.agent import _CudaBuf
    obs_dim, act_dim, B, params = SAC_CASES[case]
    ag, L = _make_learner(obs_dim, act_dim, B, params, seed)
    b = _sac_batch(obs_dim, act_dim, B, params, seed)
    args = _phase_args(b)
    assert L.lib.b2q_sac_phase(L.h, 0, *args, L._stream()) == 0
    assert L.lib.b2q_sac_phase(L.h, 2, *args, L._stream()) == 0
    dev, _ = _dev_grads(L)
    losses = torch.as_tensor(_CudaBuf(L.lib.b2q_sac_loss_ptr(L.h), 2), device="cuda").double().clone()
    p, b64 = R.to64(ag.params), _b64(b)
    dev_fw = _phase2_q(L, b["obs"], _phase2_forward(L, b["obs"], b["eps_cur"]))
    ref = {}
    for mode in ("mirror", "exact"):
        ref[mode] = R.sac_step(p, p, b64["obs"], b64["act"], b64["rew"], b64["nobs"], b64["term"], b64["eps_next"], b64["eps_cur"], GAMMA, ALPHA, mode,
                               dev=dev_fw if mode == "mirror" else None)
    m = _compare(dev, ref["mirror"][2], ref["exact"][2], ref["exact"][0])
    for i, name in enumerate(("critic_loss", "actor_loss")):
        lm, le = float(ref["mirror"][i]), float(ref["exact"][i])
        m[name] = (abs(float(losses[i]) - lm) / max(abs(lm), 1e-3), abs(float(losses[i]) - le) / max(abs(le), 1e-3), 1.0)
    L.close()
    return m


def _assert_metrics(m, tol_mirror, tol_exact=None, cos_exact=None):
    for k, (rm, re_, c) in m.items():
        loss = k.endswith("_loss")
        tm = TOL_LOSS_MIRROR if loss else tol_mirror
        assert rm < tm, (k, "mirror", rm)
        if tol_exact is not False:
            assert re_ < (tol_exact or (TOL_LOSS_EXACT if loss else TOL_EXACT)), (k, "exact", re_)
            assert loss or c > (cos_exact or COS_EXACT), (k, "exact cos", c)


@pytest.mark.parametrize("case", sorted(SAC_CASES))
def test_sac_gradients_per_tensor_vs_float64(case):
    """Every parameter tensor's gradient and both losses of phases 0 + 2, against the mirror (tight) and the exact gradient (bf16 bound)."""
    _assert_metrics(sac_case_metrics(case, 0), TOL_MIRROR[case])


def _adam_err(p_dev, p_prev, g, m, v, t, lr):
    """Adam in float64 from the device's previous parameters and its own gradient; error in units of (f32 ulp of the parameter + 1e-6 lr)."""
    import torch
    p_ref, m, v = R.adam(p_prev.double(), g.double(), m, v, t, lr)
    unit = p_ref.abs() * 2.0 ** -23 + 1e-6 * lr
    return float(((p_dev.double() - p_ref).abs() / unit).max()), m, v


def _polyak_err(t_dev, t_prev, src, tau):
    ref = R.polyak(t_prev.double(), src.double(), tau)
    return float(((t_dev.double() - ref).abs() / (ref.abs() * 2.0 ** -23 + 1e-12)).max())


TOL_ADAM_ULP = 16.0        # measured 3.5
TOL_POLYAK_ULP = 6.0       # measured 1.3
# With the device's own routing and clamp decisions fed to the mirror.  Deciding the routing in float64 instead flips one row of case c
# (third step of seed 2: a near-tie of q1 and q2 at |Q| ~ 300) and moves actor l2.weight by 1.0e-2.
TOL_LEARN_MIRROR = {"c": 4e-3,    # measured 1.0e-3 (critic l2.weight)
                    "e": 2e-3}    # measured 5.1e-4 (critic l1.weight)


def learn_order_metrics(case, seed, steps=3, feed=("a", "q", "raw_ls")):
    """learn() (critic step, then the actor gradient against the UPDATED critic, actor step, Polyak), `steps` times: per-tensor mirror error of
    both gradients the bucket holds after each call, and the Adam / Polyak error of the parameters the device produced from them.  feed: which
    of the device's phase-2 forward values the mirror takes (nets_ref.actor_step); "flips" counts the rows whose min-critic routing and the
    elements whose clamp mask the float64 mirror would have decided differently (reported, not asserted)."""
    import torch
    obs_dim, act_dim, B, params = SAC_CASES[case]
    ag, L = _make_learner(obs_dim, act_dim, B, params, seed)
    ma = va = mc = vc = 0.0
    worst = {"adam": 0.0, "polyak": 0.0}
    flips = {"route": 0, "clamp": 0}
    for t in range(1, steps + 1):
        b = _sac_batch(obs_dim, act_dim, B, params, 10 * seed + t)
        p0, tg0, (a0, c0, t0) = _state(L)
        dev_fw = _phase2_forward(L, b["obs"], b["eps_cur"])      # the actor is not stepped before phase 2
        L.learn(b["obs"], b["act"], b["rew"], b["nobs"], b["term"], eps_next=b["eps_next"], eps_cur=b["eps_cur"], pull=False)
        dev, (ga, gc) = _dev_grads(L)
        p1, _, (a1, c1, t1) = _state(L)
        b64 = _b64(b)
        _, gcm = R.critic_step(R.to64(p0), R.to64(tg0), b64["obs"], b64["act"], b64["rew"], b64["nobs"], b64["term"], b64["eps_next"], GAMMA, ALPHA, "mirror")
        _phase2_q(L, b["obs"], dev_fw)                           # after learn(): the critics phase 2 scored against
        _, gam = R.actor_step(R.to64(p0), b64["obs"], b64["eps_cur"], ALPHA, "mirror", critic=R.to64(p1), dev={k: dev_fw[k] for k in feed})
        gcm.update(gam)
        fw = R.mlp_forward(R.actor_net(R.to64(p0)), b64["obs"], act_dim, b64["eps_cur"], bf16=True)
        xin = torch.cat([b64["obs"], dev_fw["a"].double()], 1)
        q = [R.mlp_forward(R.critic_net(R.to64(p1), i), xin, bf16=True)["y"][:, 0] for i in range(2)]
        clamp = lambda r: (r > R.LOG_SIG_MIN) & (r < R.LOG_SIG_MAX)
        flips["route"] += int(((q[0] <= q[1]) != (dev_fw["q"][0] <= dev_fw["q"][1])).sum())
        flips["clamp"] += int((clamp(fw["raw_ls"]) != clamp(dev_fw["raw_ls"].double())).sum())
        for k in gcm:
            worst["grad " + k] = max(worst.get("grad " + k, 0.0), _rel(dev[k].double(), gcm[k]))
        e, ma, va = _adam_err(a1, a0, ga, ma, va, t, LR_A)
        worst["adam"] = max(worst["adam"], e)
        e, mc, vc = _adam_err(c1, c0, gc, mc, vc, t, LR_C)
        worst["adam"] = max(worst["adam"], e)
        worst["polyak"] = max(worst["polyak"], _polyak_err(t1, t0, c1, TAU))
    L.close()
    return worst, flips


@pytest.mark.parametrize("case", ["c", "e"])
def test_learn_exact_order_per_tensor_and_adam(case):
    w, flips = learn_order_metrics(case, 0)
    print(case, "decisions the float64 mirror would have flipped:", flips)
    for k, v in w.items():
        tol = TOL_ADAM_ULP if k == "adam" else TOL_POLYAK_ULP if k == "polyak" else TOL_LEARN_MIRROR[case]
        assert v < tol, (k, v)


def optimiser_metrics(seed):
    """The flat phase order (0, 2, 1, 3) for steps 1-3, then one learn(graph=True): the parameters the device produced against float64 Adam /
    Polyak applied to the device's own gradient bucket (m and v tracked here)."""
    import torch
    from paddlerobotics_b200.agent import SACLearner
    obs_dim, act_dim, B, params = SAC_CASES["a"]
    ag, L = _make_learner(obs_dim, act_dim, B, params, seed, sync="flat")
    ma = va = mc = vc = 0.0
    worst = {"adam": 0.0, "polyak": 0.0}
    for t in range(1, 5):
        b = _sac_batch(obs_dim, act_dim, B, params, 10 * seed + t)
        _, _, (a0, c0, t0) = _state(L)
        L.learn(b["obs"], b["act"], b["rew"], b["nobs"], b["term"], eps_next=b["eps_next"], eps_cur=b["eps_cur"], pull=False, graph=(t == 4))
        _, (ga, gc) = _dev_grads(L)
        _, _, (a1, c1, t1) = _state(L)
        e, ma, va = _adam_err(a1, a0, ga, ma, va, t, LR_A)
        worst["adam"] = max(worst["adam"], e)
        e, mc, vc = _adam_err(c1, c0, gc, mc, vc, t, LR_C)
        worst["adam"] = max(worst["adam"], e)
        worst["polyak"] = max(worst["polyak"], _polyak_err(t1, t0, c1, TAU))
    L.close()
    return worst


def test_optimiser_steps_are_float64_adam_and_polyak():
    """Bias-correction step index, betas, eps, both learning rates, tau and the device step counter across eager steps and a graph replay."""
    w = optimiser_metrics(0)
    assert w["adam"] < TOL_ADAM_ULP and w["polyak"] < TOL_POLYAK_ULP, w


BC_CASES = {"46of49": (49, 46, 12, 256), "20of23": (23, 20, 7, 384)}
TOL_BC_MIRROR = 1.5e-3     # measured 3.5e-4 (critic l5.bias, 46 of 49)


def bc_metrics(case, seed):
    """bc_learn: the actor gradient at the initial parameters, the critic gradient after the actor step (sampled from the updated actor)."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    ref_dim, obs_dim, act_dim, B = BC_CASES[case]
    expert, student = MujocoAgent(ref_dim, act_dim, seed=200 + seed), MujocoAgent(obs_dim, act_dim, seed=300 + seed)
    L = SACLearner(student, B, actor_lr=LR_A, critic_lr=LR_C)
    g = torch.Generator(device="cuda"); g.manual_seed(400 + seed)
    ref_obs = torch.randn(B, ref_dim, device="cuda", generator=g)
    obs = ref_obs[:, ref_dim - obs_dim:].contiguous()
    eps = torch.randn(B, act_dim, device="cuda", generator=g)
    p0 = R.to64(student.params)
    L.bc_learn(obs, ref_obs, expert, eps=eps)           # pulls the updated parameters into student.params
    dev, _ = _dev_grads(L)
    p1, pe = R.to64(student.params), R.to64(expert.params)
    o64, r64, e64 = obs.double(), ref_obs.double(), eps.double()
    ref = {}
    for mode in ("mirror", "exact"):
        bf16 = mode == "mirror"
        ref_action = R.mlp_forward(R.actor_net(pe), r64, act_dim, bf16=bf16)["predict"]
        _, ga = R.bc_actor_step(p0, o64, ref_action, mode)
        a_now = R.mlp_forward(R.actor_net(p1), o64, act_dim, e64, bf16)["sample"]
        tq = [R.mlp_forward(R.critic_net(pe, i), torch.cat([r64, a_now], 1), bf16=bf16)["y"][:, 0] for i in range(2)]
        cl, gc = R.bc_critic_step(p0, o64, a_now, tq, mode)
        gc.update(ga)
        ref[mode] = gc
    L.close()
    return _compare(dev, ref["mirror"], ref["exact"], cl)


@pytest.mark.parametrize("case", sorted(BC_CASES))
def test_bc_learn_gradients_per_tensor(case):
    _assert_metrics(bc_metrics(case, 0), tol_mirror=TOL_BC_MIRROR)
