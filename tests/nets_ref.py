"""Float64 reference of the fused MLP forward (csrc/b2q_mlp.cu) and of the SAC / behaviour-cloning learner steps (csrc/b2q_sac.cu).

Test-only.  Everything is plain torch float64 on whatever device the inputs live on, with the 3-layer backward written out by hand so that
every parameter tensor's gradient can be compared on its own.  Two modes:

  exact   no rounding anywhere: the true gradient of ETGRL/alg/sac.py:77-118 (and alg/BC.py:53-72);
  mirror  float64 arithmetic, but rounded to bf16 at exactly the points where the device rounds (operand images, activation dumps,
          the bf16 gradient tiles the tensor-core GEMMs read).  Its distance from the device measures the kernels' own arithmetic
          (f32 accumulation order, split-K atomics), so it can be held to a much tighter bound than the exact one.

Where the device rounds (read off the kernels):
  forward, every net      x, W1, W2, W3 (operand images) and h1, h2 (after bias + ReLU in f32); biases and heads stay f32
  critic head backward    dq f32; dW3 = sum dq h2; db3 = sum dq; dh2 = bf16(dq W3) . [h2 > 0] with the f32 W3 parameters; db2 = sum dh2
  hidden layers           dW2 = dh2^T h1; dh1 = bf16((dh2 W2_bf16) . [h1 > 0]); db1 = sum dh1; dW1 = dh1^T x_bf16
  dQ/da (forward_ex da)   bf16(W3_bf16 . [h2 > 0]) W2_bf16, . [h1 > 0], bf16, then . W1[:, act]_bf16
  actor head backward     dy formed in f32, rounded to bf16; db3 = sum dy; dW3 = dy^T h2; dh2 = bf16((dy W3_bf16) . [h2 > 0])
"""
import numpy as np
import torch

LOG_SIG_MAX, LOG_SIG_MIN = 2.0, -20.0
HALF_LOG_2PI = 0.9189385332046727
ACTOR = ("actor_model.l1", "actor_model.l2")
CRITICS = (("critic_model.l1", "critic_model.l2", "critic_model.l3"), ("critic_model.l4", "critic_model.l5", "critic_model.l6"))


def bf(t, on=True):
    """Round to bf16 (round-to-nearest-even, from the f32 value the device holds) and back to float64."""
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float64) if on else t


def to64(p):
    return {k: v.detach().to(torch.float64) for k, v in p.items()}


def actor_net(p):
    """(W1, b1, W2, b2, W3, b3) of the actor with W3 / b3 = cat(mean_linear, std_linear), as the kernel packs it."""
    return (p["actor_model.l1.weight"], p["actor_model.l1.bias"], p["actor_model.l2.weight"], p["actor_model.l2.bias"],
            torch.cat([p["actor_model.mean_linear.weight"], p["actor_model.std_linear.weight"]], 0),
            torch.cat([p["actor_model.mean_linear.bias"], p["actor_model.std_linear.bias"]], 0))


def critic_net(p, i):
    l1, l2, l3 = CRITICS[i]
    return tuple(p["%s.%s" % (k, s)] for k in (l1, l2, l3) for s in ("weight", "bias"))


# ---------------------------------------------------------------------------------------------------------------------------------
# forward

def mlp_layers(net, x, bf16=False):
    """One 3-layer net on input x [M, in]: returns (x as the kernel sees it, h1, h2, y) with y the pre-activation head."""
    w1, b1, w2, b2, w3, b3 = net
    r = lambda t: bf(t, bf16)
    xr = r(x)
    h1 = r(torch.relu(xr @ r(w1).T + b1))
    h2 = r(torch.relu(h1 @ r(w2).T + b2))
    return xr, h1, h2, h2 @ r(w3).T + b3


def actor_head(y, A, eps=None):
    """sac.py:60-75 on the pre-activation head y = [mean | raw log-std]: tanh(mean); with eps also the rsample() action and its log-prob."""
    mean, rl = y[:, :A], y[:, A:2 * A]
    ls = rl.clamp(LOG_SIG_MIN, LOG_SIG_MAX)
    out = dict(mean=mean, raw_ls=rl, ls=ls, predict=torch.tanh(mean))
    if eps is not None:
        x = mean + ls.exp() * eps
        a = torch.tanh(x)
        out["x_t"], out["sample"] = x, a
        out["logp"] = (-0.5 * eps * eps - ls - HALF_LOG_2PI - torch.log((1 - a * a) + 1e-6)).sum(1)
    return out


def mlp_forward(net, x, A=None, eps=None, bf16=False):
    """Forward of one net: dict with the head y and, for an actor (A given), tanh(mean) and, with eps, sample and log-prob."""
    xr, h1, h2, y = mlp_layers(net, x, bf16)
    out = dict(x=xr, h1=h1, h2=h2, y=y)
    if A is not None:
        out.update(actor_head(y, A, eps))
    return out


def dq_da(net, x, a_off, A, bf16=False):
    """dQ/da of one critic net at input x: the gradient of its scalar output wrt input columns a_off .. a_off + A - 1 ([M, A])."""
    w1, b1, w2, b2, w3, b3 = net
    r = lambda t: bf(t, bf16)
    _, h1, h2, _ = mlp_layers(net, x, bf16)
    g2 = r(r(w3)[0][None, :] * (h2 > 0))
    g1 = r((g2 @ r(w2)) * (h1 > 0))
    return g1 @ r(w1[:, a_off:a_off + A])


# ---------------------------------------------------------------------------------------------------------------------------------
# backward

def _hidden_backward(dh2, h1, x, w2, bf16):
    """Layers 2 and 1 given dh2 (already rounded where the device rounds): (dW2, db1, dW1)."""
    dW2 = dh2.T @ h1
    dh1 = bf((dh2 @ bf(w2, bf16)) * (h1 > 0), bf16)
    return dW2, dh1.sum(0), dh1.T @ x


def critic_net_grads(net, fw, dq, bf16):
    """One critic's gradients from dq [B] (dloss/dq) and its forward record fw: (W1, b1, W2, b2, W3, b3)."""
    w1, b1, w2, b2, w3, b3 = net
    dW3 = (dq @ fw["h2"])[None, :]
    db3 = dq.sum()[None]
    dh2 = bf(dq[:, None] * w3[0][None, :] * (fw["h2"] > 0), bf16)      # the head backward multiplies by the f32 parameters
    dW2, db1, dW1 = _hidden_backward(dh2, fw["h1"], fw["x"], w2, bf16)
    return dW1, db1, dW2, dh2.sum(0), dW3, db3


def actor_net_grads(net, fw, dy, bf16):
    """The actor's gradients from dy = dloss/d[mean | raw log-std] (already rounded where the device rounds)."""
    w1, b1, w2, b2, w3, b3 = net
    dW3 = dy.T @ fw["h2"]
    dh2 = bf((dy @ bf(w3, bf16)) * (fw["h2"] > 0), bf16)
    dW2, db1, dW1 = _hidden_backward(dh2, fw["h1"], fw["x"], w2, bf16)
    return dW1, db1, dW2, dh2.sum(0), dW3, dy.sum(0)


def _named_actor(g, A):
    dW1, db1, dW2, db2, dW3, db3 = g
    return {"actor_model.l1.weight": dW1, "actor_model.l1.bias": db1, "actor_model.l2.weight": dW2, "actor_model.l2.bias": db2,
            "actor_model.mean_linear.weight": dW3[:A], "actor_model.std_linear.weight": dW3[A:],
            "actor_model.mean_linear.bias": db3[:A], "actor_model.std_linear.bias": db3[A:]}


def _named_critic(g, i):
    return {"%s.%s" % (k, s): t for (k, s), t in zip([(k, s) for k in CRITICS[i] for s in ("weight", "bias")], g)}


def critic_step(p, tgt, obs, act, rew, nobs, term, eps_next, gamma, alpha, mode="exact"):
    """The critic half of SAC.learn (sac.py:85-96): (critic_loss, {critic tensor name: gradient}).  p: actor + critics, tgt: target critics."""
    bf16 = mode == "mirror"
    A = act.shape[1]
    nxt = mlp_forward(actor_net(p), nobs, A, eps_next, bf16)
    na = nxt["sample"]
    qn = [mlp_forward(critic_net(tgt, i), torch.cat([nobs, na], 1), bf16=bf16)["y"][:, 0] for i in range(2)]
    tq = rew + gamma * term * (torch.minimum(qn[0], qn[1]) - alpha * nxt["logp"])
    B = obs.shape[0]
    loss, grads = 0.0, {}
    for i in range(2):
        net = critic_net(p, i)
        fw = mlp_forward(net, torch.cat([obs, act], 1), bf16=bf16)
        e = fw["y"][:, 0] - tq
        loss = loss + (e * e).mean()
        grads.update(_named_critic(critic_net_grads(net, fw, 2 * e / B, bf16), i))
    return loss, grads


def actor_step(p, obs, eps_cur, alpha, mode="exact", critic=None, dev=None):
    """The actor half of SAC.learn (sac.py:102-110): (actor_loss, {actor tensor name: gradient}).  critic: the parameters the actor is
    scored against (default p itself; learn() uses the critics after their optimiser step).

    dev (mirror): what the device's own f32 forward produced, used in place of the reference's float64 values where a last-bit difference
    does not stay small:  "a", the sampled actions (on saturated actions one ulp of a moves 1 - a^2 by 1.2e-7, which the log(1 - a^2 + 1e-6)
    term amplifies up to 1e6-fold);  "q" = (q1, q2) at those actions, which decide where d min(q1, q2)/da goes;  "raw_ls", the raw log-std,
    which decides the clamp mask.  A near-tie on either of the last two flips a whole element of dy."""
    bf16 = mode == "mirror"
    critic = p if critic is None else critic
    dev = dev or {}
    B, A = eps_cur.shape
    D = obs.shape[1]
    net = actor_net(p)
    fw = mlp_forward(net, obs, A, eps_cur, bf16)
    f64 = lambda t: t.to(fw["y"])
    a, sd = (f64(dev["a"]) if "a" in dev else fw["sample"]), fw["ls"].exp()
    xin = torch.cat([obs, a], 1)
    q = [mlp_forward(critic_net(critic, i), xin, bf16=bf16)["y"][:, 0] for i in range(2)]
    da = [dq_da(critic_net(critic, i), xin, D, A, bf16) for i in range(2)]
    loss = (alpha * fw["logp"] - torch.minimum(q[0], q[1])).mean()
    qr = [f64(t) for t in dev["q"]] if "q" in dev else q
    rl = f64(dev["raw_ls"]) if "raw_ls" in dev else fw["raw_ls"]
    dqa = torch.where((qr[0] <= qr[1])[:, None], da[0], da[1])                # torch.min routes ties to the first argument
    ga = -dqa / B + (alpha / B) * (2 * a / ((1 - a * a) + 1e-6))
    gx = ga * (1 - a * a)
    gls = (gx * sd * eps_cur - alpha / B) * ((rl > LOG_SIG_MIN) & (rl < LOG_SIG_MAX))
    dy = bf(torch.cat([gx, gls], 1), bf16)
    return loss, _named_actor(actor_net_grads(net, fw, dy, bf16), A)


def sac_step(p, tgt, obs, act, rew, nobs, term, eps_next, eps_cur, gamma, alpha, mode="exact", critic_for_actor=None, dev=None):
    """Both halves: (critic_loss, actor_loss, {every parameter tensor: gradient}).  Without critic_for_actor both gradients are taken at the
    same parameters (the flat phase order 0, 2); with it the actor is scored against those critics (learn(): the updated ones).  dev: see
    actor_step."""
    cl, g = critic_step(p, tgt, obs, act, rew, nobs, term, eps_next, gamma, alpha, mode)
    al, ga = actor_step(p, obs, eps_cur, alpha, mode, critic_for_actor, dev)
    g.update(ga)
    return cl, al, g


def bc_actor_step(p, obs, ref_action, mode="exact"):
    """BC.py:53-59: actor_loss = -mean log N(ref_action | mean, exp(log_std)) and the actor gradients."""
    bf16 = mode == "mirror"
    B, A = ref_action.shape
    net = actor_net(p)
    fw = mlp_forward(net, obs, A, None, bf16)
    d, ls, rl = ref_action - fw["mean"], fw["ls"], fw["raw_ls"]
    iv = torch.exp(-2 * ls)
    loss = -(-0.5 * d * d * iv - ls - HALF_LOG_2PI).mean()
    g0 = -(d * iv) / (B * A)
    g1 = -(d * d * iv - 1) / (B * A) * ((rl > LOG_SIG_MIN) & (rl < LOG_SIG_MAX))
    dy = bf(torch.cat([g0, g1], 1), bf16)
    return loss, _named_actor(actor_net_grads(net, fw, dy, bf16), A)


def bc_critic_step(p, obs, a_now, target_q, mode="exact"):
    """BC.py:61-72: critic regression of Q_i(obs, a_now) onto target_q[i]: (critic_loss, critic gradients)."""
    bf16 = mode == "mirror"
    B = obs.shape[0]
    loss, grads = 0.0, {}
    for i in range(2):
        net = critic_net(p, i)
        fw = mlp_forward(net, torch.cat([obs, a_now], 1), bf16=bf16)
        e = fw["y"][:, 0] - target_q[i]
        loss = loss + (e * e).mean()
        grads.update(_named_critic(critic_net_grads(net, fw, 2 * e / B, bf16), i))
    return loss, grads


# ---------------------------------------------------------------------------------------------------------------------------------
# optimiser

def adam(p, g, m, v, t, lr, b1=0.9, b2=0.999, eps=1e-8):
    """torch.optim.Adam (defaults, no weight decay) step number t in float64 (sac.py:55-58); returns (p, m, v)."""
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    return p - lr / (1 - b1 ** t) * m / ((v / (1 - b2 ** t)).sqrt() + eps), m, v


def polyak(tgt, src, tau):
    """sync_target (sac.py:112-118)."""
    return tau * src + (1 - tau) * tgt


# ---------------------------------------------------------------------------------------------------------------------------------
# counter RNG (b2q_philox.cuh)

GOLDEN_GAMMA = 0x9E3779B97F4A7C15
_M32 = np.uint64(0xFFFFFFFF)


def effective_seed(seed, ctr):
    """The sampling key of a launch whose device-side step counter reads ctr."""
    return (int(seed) + (int(ctr) & 0xFFFFFFFF) * GOLDEN_GAMMA) % (1 << 64)


def philox_normal(seed, row, col):
    """N(0, 1) draw of element (row, col) under a 64-bit key: Philox-4x32-10 with counter (row, col, 0x9E3779B9, 0), Box-Muller of the top 24
    bits of the first two words.  The product 2 pi u2 is rounded to f32 as the device forms it; the rest is float64.  Broadcasts row / col."""
    row, col = np.broadcast_arrays(np.asarray(row, np.uint64), np.asarray(col, np.uint64))
    c0, c1 = row & _M32, col & _M32
    c2 = np.full(c0.shape, 0x9E3779B9, np.uint64)
    c3 = np.zeros(c0.shape, np.uint64)
    seed = int(seed) % (1 << 64)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2            # 32 x 32 -> 64-bit products: (mulhi, mullo)
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & _M32
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    # the uniforms as the device forms them: (float)(c >> 8) + 0.5f rounds to 24 bits, the scale by 2^-24 is exact
    u = [((c >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0) for c in (c0, c1)]
    arg = (np.float32(6.283185307179586) * u[1]).astype(np.float64)
    return np.sqrt(-2.0 * np.log(u[0].astype(np.float64))) * np.cos(arg)


def philox_eps(seed, B, A):
    """[B, A] float32 draws of rows 0..B-1, actions 0..A-1 under key seed."""
    return philox_normal(seed, np.arange(B)[:, None], np.arange(A)[None, :]).astype(np.float32)
