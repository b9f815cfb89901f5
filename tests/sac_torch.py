"""A plain torch restatement of ETGRL/alg/sac.py:77-118 (autograd-able, any dtype, any device): the yardstick the SAC tests differentiate
with torch.autograd.  Shared by the GPU learner tests and the CPU self-check of the float64 reference (tests/nets_ref.py)."""


def torch_sac_losses(p, tgt, obs, act, rew, nobs, term, eps_next, eps_cur, gamma, alpha):
    """(critic_loss, actor_loss), both at the parameters p (no critic update in between); eps_next / eps_cur are the fixed N(0, 1) draws of
    the two rsample() calls.  Differentiate them with torch.autograd."""
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
