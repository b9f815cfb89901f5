"""K5/K6: SAC.learn on the device vs a plain PyTorch fp32 restatement of ETGRL/alg/sac.py:77-118 (same minibatch, same
N(0,1) draws for both rsample() calls).  Forward/backward GEMMs run in bf16 on wgmma tensor cores with f32 accumulation, so the
tolerance is the bf16 one: losses within 2 %, gradient buckets within 5 % relative L2 error and cosine >= 0.995."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _torch_sac_step(p, tgt, obs, act, rew, nobs, term, eps_next, eps_cur, gamma, alpha):
    """Returns critic_loss, actor_loss and gradients w.r.t. every parameter (critic grads from the critic loss, actor
    grads from the actor loss evaluated AFTER the critic update is skipped — i.e. both at the same parameters)."""
    import torch
    import torch.nn.functional as F

    def actor(pp, o):
        x = F.relu(F.linear(o, pp["actor_model.l1.weight"], pp["actor_model.l1.bias"]))
        x = F.relu(F.linear(x, pp["actor_model.l2.weight"], pp["actor_model.l2.bias"]))
        mean = F.linear(x, pp["actor_model.mean_linear.weight"], pp["actor_model.mean_linear.bias"])
        ls = torch.clamp(F.linear(x, pp["actor_model.std_linear.weight"], pp["actor_model.std_linear.bias"]), -20.0, 2.0)
        return mean, ls

    def critic(pp, o, a):
        x = torch.cat([o, a], 1)
        out = []
        for l1, l2, l3 in (("l1", "l2", "l3"), ("l4", "l5", "l6")):
            h = F.relu(F.linear(x, pp["critic_model.%s.weight" % l1], pp["critic_model.%s.bias" % l1]))
            h = F.relu(F.linear(h, pp["critic_model.%s.weight" % l2], pp["critic_model.%s.bias" % l2]))
            out.append(F.linear(h, pp["critic_model.%s.weight" % l3], pp["critic_model.%s.bias" % l3]))
        return out

    def sample(pp, o, eps):
        mean, ls = actor(pp, o)
        std = ls.exp()
        x_t = mean + std * eps                                              # rsample with a fixed draw
        a = torch.tanh(x_t)
        logp = torch.distributions.Normal(mean, std).log_prob(x_t) - torch.log((1 - a.pow(2)) + 1e-6)
        return a, logp.sum(1, keepdim=True)

    with torch.no_grad():
        na, nlp = sample(p, nobs, eps_next)
        q1n, q2n = critic(tgt, nobs, na)
        target_q = rew[:, None] + gamma * term[:, None] * (torch.min(q1n, q2n) - alpha * nlp)
    q1, q2 = critic(p, obs, act)
    critic_loss = F.mse_loss(q1, target_q) + F.mse_loss(q2, target_q)
    a, lp = sample(p, obs, eps_cur)
    q1p, q2p = critic(p, obs, a)
    actor_loss = (alpha * lp - torch.min(q1p, q2p)).mean()
    return critic_loss, actor_loss


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


def test_counter_rng_noise_is_the_same_draw_in_forward_and_backward():
    """eps = None: both rsample() draws come from the counter RNG inside the kernels.  The backward must differentiate through the SAME draw the
    forward used: recover the draws from the forward's outputs (fresh learner: step counter 0, so the key is the host seed alone), feed them
    back as explicit eps to a second learner and compare the gradients."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner, SAMPLE
    B, seed = 256, 7
    g = torch.Generator(device="cuda"); g.manual_seed(31)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    obs, nobs, act, rew, term = r(B, 49), r(B, 49), torch.rand(B, 12, device="cuda", generator=g) * 2 - 1, r(B), torch.ones(B, device="cuda")
    grads = []
    eps = [None, None]
    for explicit in (False, True):
        ag = MujocoAgent(49, 12, seed=17)
        L = SACLearner(ag, B)
        if not explicit:   # the draws of element (row, col) under keys 2*seed (current obs) and 2*seed + 1 (next obs), from the sampled actions
            for k, (o, sd) in enumerate(((nobs, 2 * seed + 1), (obs, 2 * seed))):
                a, _, raw = L.actor.forward(o, mode=SAMPLE, seed=sd, want_raw=True)
                mean, ls = raw[0, :, :12], raw[0, :, 12:].clamp(-20, 2)
                eps[k] = ((torch.atanh(a[0].double().clamp(-1 + 1e-12, 1 - 1e-12)) - mean.double()) / ls.double().exp()).float()
            assert 0.9 < float(eps[0].std()) < 1.1 and abs(float(eps[0].mean())) < 0.1
        pe = lambda x: x.data_ptr() if explicit else None
        args = (obs.data_ptr(), act.data_ptr(), rew.data_ptr(), nobs.data_ptr(), term.data_ptr(), pe(eps[0]), pe(eps[1]), seed)
        assert L.lib.b2q_sac_phase(L.h, 0, *args, L._stream()) == 0
        assert L.lib.b2q_sac_phase(L.h, 2, *args, L._stream()) == 0
        grads.append([x.clone() for x in L.grads()])
        torch.cuda.synchronize()
    for x, y in zip(grads[0], grads[1]):
        cos = float(torch.dot(x, y) / (x.norm() * y.norm()))
        rel = float((x - y).norm() / y.norm())
        print("counter-RNG vs explicit eps: cos %.6f rel %.4g" % (cos, rel))
        assert cos > 0.9995 and rel < 0.03, (cos, rel)     # atanh of a saturated f32 action limits how exactly the draw can be recovered


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
