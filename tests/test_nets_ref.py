"""The float64 reference of tests/nets_ref.py checked against torch.autograd, without a GPU: the hand-written backward in `exact` mode
is the true gradient of sac.py:77-118 / BC.py:53-72 (to 2e-9) at every learner shape the GPU tests use, and `mirror` differs from it
only by its bf16 rounding points."""
import numpy as np
import pytest
import torch

import nets_ref as R
from sac_torch import torch_sac_losses as _torch_sac_step

SHAPES = [(49, 12), (46, 12), (52, 12), (3, 1), (20, 7)]


def _params(obs_dim, act_dim, seed):
    """State dict of a fresh agent (nn.Linear init), float64; actions 0, 1 of the log-std head pushed into the lower clamp and 2, 3 into
    the upper one where there are enough actions (the clamp-gradient mask)."""
    g = torch.Generator().manual_seed(seed)
    shapes = [("actor_model.l1", 256, obs_dim), ("actor_model.l2", 256, 256), ("actor_model.mean_linear", act_dim, 256),
              ("actor_model.std_linear", act_dim, 256)]
    for net in R.CRITICS:
        shapes += [(net[0], 256, obs_dim + act_dim), (net[1], 256, 256), (net[2], 1, 256)]
    p = {}
    for name, o, i in shapes:
        bound = 1.0 / np.sqrt(i)
        p[name + ".weight"] = ((torch.rand(o, i, generator=g, dtype=torch.float64) * 2 - 1) * bound)
        p[name + ".bias"] = ((torch.rand(o, generator=g, dtype=torch.float64) * 2 - 1) * bound)
    if act_dim >= 4:
        p["actor_model.std_linear.bias"][:2] = -25.0
        p["actor_model.std_linear.bias"][2:4] = 3.0
    return p


def _batch(obs_dim, act_dim, B, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    return dict(obs=r(B, obs_dim), act=torch.rand(B, act_dim, generator=g, dtype=torch.float64) * 2 - 1, rew=r(B), nobs=r(B, obs_dim),
                term=(torch.rand(B, generator=g, dtype=torch.float64) > 0.1).double(), eps_next=r(B, act_dim), eps_cur=r(B, act_dim))


def _close(got, ref, tol=2e-9):
    """Max error relative to the tensor's largest entry.  2e-9 rather than float64's 1e-15: on saturated actions d log(1 - a^2 + 1e-6)/da
    multiplies the rounding of 1 - a^2 by up to 1e6, so two correct float64 evaluations of the actor gradient differ by up to 8e-10."""
    for k, r in ref.items():
        err = float((got[k] - r).abs().max()) / max(1.0, float(r.abs().max()))
        assert err < tol, (k, err)


@pytest.mark.parametrize("obs_dim,act_dim", SHAPES)
def test_exact_backward_is_the_autograd_gradient(obs_dim, act_dim):
    p = _params(obs_dim, act_dim, obs_dim)
    tgt = {k: v + 0.01 * torch.randn_like(v) for k, v in p.items()}
    b = _batch(obs_dim, act_dim, 96, act_dim)
    gamma, alpha = 0.99, 0.2
    pg = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    cl, al = _torch_sac_step(pg, tgt, b["obs"], b["act"], b["rew"], b["nobs"], b["term"], b["eps_next"], b["eps_cur"], gamma, alpha)
    ck = [k for k in p if k.startswith("critic")]
    ak = [k for k in p if k.startswith("actor")]
    ref = dict(zip(ck, torch.autograd.grad(cl, [pg[k] for k in ck], retain_graph=True)))
    ref.update(zip(ak, torch.autograd.grad(al, [pg[k] for k in ak])))
    c, a, g = R.sac_step(p, tgt, b["obs"], b["act"], b["rew"], b["nobs"], b["term"], b["eps_next"], b["eps_cur"], gamma, alpha, "exact")
    assert abs(float(c) - float(cl.detach())) < 1e-10 * max(1.0, abs(float(cl.detach())))
    assert abs(float(a) - float(al.detach())) < 1e-10 * max(1.0, abs(float(al.detach())))
    assert set(g) == set(p)
    _close(g, ref)
    if act_dim >= 4:      # always-clamped log-std actions get no gradient at all
        for k in ("actor_model.std_linear.weight", "actor_model.std_linear.bias"):
            assert float(g[k][:4].abs().max()) == 0.0


@pytest.mark.parametrize("obs_dim,act_dim", [(49, 12), (20, 7)])
def test_exact_actor_step_against_given_critic_is_the_autograd_gradient(obs_dim, act_dim):
    """learn()'s order: the actor loss is scored against a different (updated) critic than the one the critic gradient was taken at."""
    p = _params(obs_dim, act_dim, 5)
    crit = {k: v + 0.02 * torch.randn_like(v) for k, v in p.items()}
    b = _batch(obs_dim, act_dim, 64, 6)
    mixed = {k: (p[k] if k.startswith("actor") else crit[k]).clone().requires_grad_(True) for k in p}
    _, al = _torch_sac_step(mixed, crit, b["obs"], b["act"], b["rew"], b["nobs"], b["term"], b["eps_next"], b["eps_cur"], 0.99, 0.2)
    ak = [k for k in p if k.startswith("actor")]
    ref = dict(zip(ak, torch.autograd.grad(al, [mixed[k] for k in ak])))
    a, g = R.actor_step(p, b["obs"], b["eps_cur"], 0.2, "exact", critic=crit)
    assert abs(float(a) - float(al.detach())) < 1e-10 * max(1.0, abs(float(al.detach())))
    _close(g, ref)


@pytest.mark.parametrize("obs_dim,act_dim", [(46, 12), (20, 7)])
def test_exact_bc_steps_are_the_autograd_gradient(obs_dim, act_dim):
    import torch.nn.functional as F
    p = _params(obs_dim, act_dim, 9)
    b = _batch(obs_dim, act_dim, 64, 10)
    ref_action = torch.tanh(b["eps_next"])
    pg = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    y = R.mlp_forward(R.actor_net(pg), b["obs"])["y"]          # the forward itself is plain autograd-able torch
    mean, ls = y[:, :act_dim], y[:, act_dim:].clamp(-20.0, 2.0)
    al = -torch.distributions.Normal(mean, ls.exp()).log_prob(ref_action).mean()
    ak = [k for k in p if k.startswith("actor")]
    ref = dict(zip(ak, torch.autograd.grad(al, [pg[k] for k in ak])))
    a, g = R.bc_actor_step(p, b["obs"], ref_action, "exact")
    assert abs(float(a) - float(al.detach())) < 1e-10 * max(1.0, abs(float(al.detach())))
    _close(g, ref)
    tq = [b["rew"], b["rew"] * 2]
    cl = sum(F.mse_loss(R.mlp_forward(R.critic_net(pg, i), torch.cat([b["obs"], b["act"]], 1))["y"][:, 0], tq[i]) for i in range(2))
    ck = [k for k in p if k.startswith("critic")]
    ref = dict(zip(ck, torch.autograd.grad(cl, [pg[k] for k in ck])))
    c, g = R.bc_critic_step(p, b["obs"], b["act"], tq, "exact")
    assert abs(float(c) - float(cl.detach())) < 1e-10 * max(1.0, abs(float(cl.detach())))
    _close(g, ref)


def test_dq_da_is_the_autograd_input_gradient():
    p = _params(20, 7, 3)
    x = torch.randn(50, 27, dtype=torch.float64, requires_grad=True)
    for i in range(2):
        net = R.critic_net(p, i)
        (gx,) = torch.autograd.grad(R.mlp_forward(net, x)["y"].sum(), [x])
        assert float((R.dq_da(net, x.detach(), 20, 7) - gx[:, 20:]).abs().max()) < 1e-12


def test_mirror_without_rounding_is_exact(monkeypatch):
    """`mirror` is `exact` plus rounding: with the rounding switched off the two agree to the last bit of float64 arithmetic."""
    p = _params(20, 7, 4)
    tgt = {k: v.clone() for k, v in p.items()}
    b = _batch(20, 7, 64, 4)
    args = (p, tgt, b["obs"], b["act"], b["rew"], b["nobs"], b["term"], b["eps_next"], b["eps_cur"], 0.99, 0.2)
    ce, ae, ge = R.sac_step(*args, mode="exact")
    cm, am, gm = R.sac_step(*args, mode="mirror")
    assert any(float((ge[k] - gm[k]).abs().max()) > 0 for k in ge)      # rounding on: the two differ
    monkeypatch.setattr(R, "bf", lambda t, on=True: t)
    cm, am, gm = R.sac_step(*args, mode="mirror")
    assert float(cm) == float(ce) and float(am) == float(ae)
    for k in ge:
        assert torch.equal(gm[k], ge[k]), k
    _, gbe = R.bc_actor_step(p, b["obs"], torch.tanh(b["eps_cur"]), "exact")
    _, gbm = R.bc_actor_step(p, b["obs"], torch.tanh(b["eps_cur"]), "mirror")
    for k in gbe:
        assert torch.equal(gbm[k], gbe[k]), k


def test_bf16_rounding_is_round_to_nearest_even():
    x = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -9, -(1.0 + 2 ** -7 + 2 ** -9)], dtype=torch.float64)
    assert R.bf(x).tolist() == [1.0, 1.0 + 2 ** -6, 1.0, -(1.0 + 2 ** -7)]
    assert torch.equal(R.bf(x, on=False), x)


def test_adam_and_polyak_follow_torch():
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(100, generator=g, dtype=torch.float64)
    w = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([w], lr=3e-4)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for t in (1, 2, 3):
        gr = torch.randn(100, generator=g, dtype=torch.float64) * 10.0 ** -t
        w.grad = gr.clone()
        opt.step()
        p, m, v = R.adam(p, gr, m, v, t, 3e-4)
        assert float((p - w.detach()).abs().max()) < 1e-15
    assert torch.equal(R.polyak(torch.zeros(3), torch.ones(3), 0.25), torch.full((3,), 0.25))


def test_philox_normal_is_a_standard_normal_and_keyed():
    e = R.philox_eps(7, 4096, 12)
    assert e.dtype == np.float32 and abs(float(e.mean())) < 0.02 and abs(float(e.std()) - 1) < 0.02
    assert np.array_equal(e, R.philox_eps(7, 4096, 12)) and not np.array_equal(e, R.philox_eps(8, 4096, 12))
    assert np.float32(R.philox_normal(7, 5, 3)) == e[5, 3]
    assert R.effective_seed(5, 0) == 5 and R.effective_seed(5, 2) == (5 + 2 * 0x9E3779B97F4A7C15) % 2 ** 64
