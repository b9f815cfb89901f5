"""K3: fused wgmma MLP forward vs a plain PyTorch fp32 reference of the same op, and vs the known answers of the
reference's shipped checkpoint (tests/golden/StairStair3_BC1_itr_500383.pt; vectors made by the unmodified
model/mujoco_model.py).  Arithmetic is bf16 x bf16 -> f32 (BASELINE: bf16 tensor-core GEMM), so the tolerance is the
bf16 one: |err| <= 2e-2 + 3e-2*max(1,|ref|) on pre-activations of the trained checkpoint (measured 4e-2 at |ref|~1.5),
<= 2e-2 on tanh outputs of fresh nets, Q values <= 1% + 0.3; against a reference with bf16-ROUNDED operands (isolating the
kernel's own f32-accumulate arithmetic) <= 2e-3."""
import ctypes as C
import os

import numpy as np
import pytest

import nets_ref as R

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


# ---------------------------------------------------------------------------------------------------------------------------------
# The forward over the ABI's range, against the float64 reference of tests/nets_ref.py: `mirror` (bf16 operands and activations where the
# kernel rounds them) isolates the kernel's own f32 arithmetic; `exact` is the plain float64 net.  Bounds are about 4x the largest value
# measured on an H100 (80GB HBM3) over seeds 0, 1, 2; the measured value is beside each.
NAN_BITS = 0x7FC0DEAD      # a quiet NaN no kernel writes: the guard regions and unwritten bodies are recognisable bit for bit
GUARD = 64
#            in1  in2  mode      out  nets  M        (mode: 0 PREDICT, 1 SAMPLE, 2 RAW)
MLP_CASES = [(1, 0, 2, 1, 1, 1),
             (3, 1, 1, 2, 1, 129),           # SAMPLE, A = 1
             (16, 0, 0, 10, 3, 127),         # PREDICT, A = 5
             (5, 12, 2, 3, 2, 128),          # odd RAW width
             (33, 0, 1, 14, 1, 4097),        # SAMPLE, A = 7
             (52, 12, 2, 1, 2, 1000),        # in_dim = 64: no zero padding in the K panel
             (64, 0, 1, 32, 8, 300),         # SAMPLE, A = 16, eight nets
             (63, 0, 2, 32, 8, 65536),
             (49, 0, 1, 24, 1, 65537)]       # the A = 12 compile-time head, a one-row last tile
TOL_Y_MIRROR = 4e-3         # max |y - y_mirror| / max(1, max |y_mirror|): measured 8.9e-4 (RAW 32, 8 nets, M 65536)
TOL_Y_EXACT = 5e-2          # relative L2 of y against the exact net: measured 1.2e-2 (in_dim 1, M 1)
TOL_OUT_MIRROR = 4e-3       # max |tanh / sample / raw - mirror|: measured 8.9e-4
TOL_LOGP_MIRROR = 8e-2      # max |logp - mirror| / (1 + sum_j 1e-6 / (1 - a_j^2 + 1e-6)): measured 2.8e-3 fresh, 2.0e-2 checkpoint
TOL_RNG_OUT, TOL_RNG_LOGP = 1e-6, 6e-4    # counter-RNG call vs the explicit numpy Philox draws: measured 2.4e-7, 1.4e-4


def _guarded(shape):
    """A float32 device buffer of `shape` followed by GUARD floats, all set to the NaN pattern: (whole buffer, body view)."""
    import torch
    n = int(np.prod(shape))
    full = torch.full((n + GUARD,), NAN_BITS, dtype=torch.int32, device="cuda").view(torch.float32)
    return full, full[:n].view(*shape)


def _check_guard(full, shape):
    import torch
    n = int(np.prod(shape))
    assert bool(torch.isfinite(full[:n]).all()), "output body not fully written"
    assert bool((full[n:].view(torch.int32) == NAN_BITS).all()), "write past the end of the output"


def _random_net(in_dim, out_dim, g):
    import torch
    net = []
    for o, i in ((256, in_dim), (256, 256), (out_dim, 256)):
        bound = 1.0 / np.sqrt(i)
        net += [((torch.rand(o, i, generator=g, device="cuda") * 2 - 1) * bound).contiguous(), (torch.rand(o, generator=g, device="cuda") * 2 - 1) * bound]
    return net


def _lp_scale(a):
    """The f32 rounding of a = tanh(x) near +-1 moves log(1 - a^2 + 1e-6) by up to ~1e-7 / (1 - a^2 + 1e-6): the log-prob's conditioning."""
    return 1 + (1e-6 / ((1 - a * a) + 1e-6)).sum(-1)


def _forward(mlp, in1, in2, mode, seed, eps, A, want_logp):
    """b2q_mlp_forward into guarded, NaN-filled buffers; checks the guards and returns (out, logp, raw)."""
    nets, M, od = mlp.nets, in1.shape[0], mlp.out_dim
    bufs = [_guarded((nets, M, A)), _guarded((nets, M)) if want_logp else None, _guarded((nets, M, od))]
    p = lambda t: None if t is None else t.data_ptr()
    rc = mlp.lib.b2q_mlp_forward(mlp.h, in1.data_ptr(), in1.shape[1], p(in2), M, mode, C.c_uint64(seed), p(eps), bufs[0][0].data_ptr(),
                                 bufs[1][0].data_ptr() if want_logp else None, bufs[2][0].data_ptr(), mlp._stream())
    assert rc == 0, mlp.lib.b2q_mlp_last_error(mlp.h)
    import torch
    torch.cuda.synchronize()
    for bf, shape in zip(bufs, [(nets, M, A), (nets, M), (nets, M, od)]):
        if bf is not None:
            _check_guard(bf[0], shape)
    return bufs[0][1], bufs[1][1] if want_logp else None, bufs[2][1]


def mlp_case_metrics(case, seed):
    import torch
    from paddlerobotics_b200.agent import FusedMLP
    in1_dim, in2_dim, mode, od, nets, M = case
    in_dim = in1_dim + in2_dim
    g = torch.Generator(device="cuda"); g.manual_seed(500 + seed)
    mlp = FusedMLP(in_dim, od, nets)
    ws = [_random_net(in_dim, od, g) for _ in range(nets)]
    for i, w in enumerate(ws):
        mlp.set_weights(i, *w)
    in1 = torch.randn(M, in1_dim, device="cuda", generator=g)
    in2 = (torch.rand(M, in2_dim, device="cuda", generator=g) * 2 - 1) if in2_dim else None
    x64 = (torch.cat([in1, in2], 1) if in2_dim else in1).double()
    A = od if mode == 2 else od // 2
    eps = None
    m = {}
    if mode == 1:
        key = 1234567 + seed
        out_c, lp_c, _ = _forward(mlp, in1, in2, mode, key, None, A, True)
        eps = torch.as_tensor(R.philox_eps(key, M, A), device="cuda")
    out, lp, raw = _forward(mlp, in1, in2, mode, 99, eps, A, mode == 1)
    m.update(y_mirror=0.0, y_exact=0.0, out_mirror=0.0, logp_mirror=0.0)
    for i in range(nets):
        net = [t.double() for t in ws[i]]
        mir = R.mlp_forward(net, x64, None if mode == 2 else A, None if eps is None else eps.double(), bf16=True)
        ex = R.mlp_forward(net, x64, bf16=False)
        y = raw[i].double()
        m["y_mirror"] = max(m["y_mirror"], float((y - mir["y"]).abs().max()) / max(1.0, float(mir["y"].abs().max())))
        m["y_exact"] = max(m["y_exact"], float((y - ex["y"]).norm() / ex["y"].norm()))
        ref_out = mir["y"] if mode == 2 else (mir["predict"] if mode == 0 else mir["sample"])
        m["out_mirror"] = max(m["out_mirror"], float((out[i].double() - ref_out).abs().max()))
        if mode == 1:
            m["logp_mirror"] = max(m["logp_mirror"], float(((lp[i].double() - mir["logp"]).abs() / _lp_scale(mir["sample"])).max()))
    if mode == 1:     # eps = None: the counter-RNG draw of element (row, col) is the numpy Philox draw
        m["rng_out"] = float((out_c - out).abs().max())
        m["rng_logp"] = float(((lp_c - lp).abs().double() / _lp_scale(out.double())).max())
    mlp.close()
    return m


def _assert_mlp(m):
    tol = dict(y_mirror=TOL_Y_MIRROR, y_exact=TOL_Y_EXACT, out_mirror=TOL_OUT_MIRROR, logp_mirror=TOL_LOGP_MIRROR, rng_out=TOL_RNG_OUT, rng_logp=TOL_RNG_LOGP)
    for k, v in m.items():
        assert v < tol[k], (k, v)


@pytest.mark.parametrize("case", MLP_CASES, ids=["in%d+%d-mode%d-out%d-nets%d-M%d" % c for c in MLP_CASES])
def test_forward_over_the_abi_range_vs_float64(case):
    """Output bodies fully written and finite, guards after them untouched; the head against the mirror (tight) and the exact net (bf16
    bound); SAMPLE with eps = None equal to the explicit call with the numpy Philox draws."""
    _assert_mlp(mlp_case_metrics(case, 0))


def checkpoint_sample_metrics(seed):
    """The shipped checkpoint at the 16 golden observations (|mean| up to 3, the upper log-std clamp on 8 of 12 actions): SAMPLE with explicit
    draws, every row's action and log-prob against the mirror."""
    import torch
    from paddlerobotics_b200.agent import MujocoAgent
    ag = MujocoAgent(46, 12)
    ag.restore(os.path.join(GOLDEN, "StairStair3_BC1_itr_500383.pt"))
    obs = torch.tensor(np.load(os.path.join(GOLDEN, "reference_vectors.npz"))["mlp_obs"], device="cuda")
    eps = torch.as_tensor(R.philox_eps(77 + seed, 16, 12), device="cuda")
    out, lp, raw = _forward(ag.actor, obs, None, 1, 0, eps, 12, True)
    mir = R.mlp_forward(R.actor_net(R.to64(ag.params)), obs.double(), 12, eps.double(), bf16=True)
    assert bool((mir["raw_ls"] > 2.0).any())          # the upper clamp is really reached
    return dict(y_mirror=float((raw[0].double() - mir["y"]).abs().max()) / max(1.0, float(mir["y"].abs().max())),
                out_mirror=float((out[0].double() - mir["sample"]).abs().max()),
                logp_mirror=float(((lp[0].double() - mir["logp"]).abs() / _lp_scale(mir["sample"])).max()))


def test_checkpoint_sample_and_logprob_vs_float64():
    _assert_mlp(checkpoint_sample_metrics(0))


DA_SHAPES = [(49, 12), (52, 12), (3, 1), (20, 7)]
TOL_DA_MIRROR = 3e-3        # relative L2 against the mirror: measured 7.4e-4 (52 + 12, M 8192)
TOL_DA_EXACT = 0.3          # relative L2 against the float64 autograd dQ/da: measured 0.072 (M >= 129)
TOL_DA_EXACT_M1 = 0.85      # one row (A numbers): measured 0.21.  Not meant to catch errors: on a single row a few ReLU-mask flips
                            # from bf16 rounding dominate; at M = 1 the mirror bound does the checking


def _forward_ex(lib):
    f = lib.b2q_mlp_forward_ex
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    s = lib.b2q_mlp_set_action_slice
    s.restype = C.c_int
    s.argtypes = [C.c_void_p, C.c_int, C.c_int]
    return f, s


def dqda_metrics(obs_dim, act_dim, M, seed):
    """dQ_i/da of both critics from b2q_mlp_forward_ex(..., da): the action columns against the mirror and the float64 autograd gradient,
    the unused columns A..15 exactly zero."""
    import torch
    from paddlerobotics_b200.agent import FusedMLP
    g = torch.Generator(device="cuda"); g.manual_seed(700 + seed)
    mlp = FusedMLP(obs_dim + act_dim, 1, 2)
    fwd_ex, set_slice = _forward_ex(mlp.lib)
    assert set_slice(mlp.h, obs_dim, act_dim) == 0         # before set_weights: the pack kernel fills the W1 action-column image
    ws = [_random_net(obs_dim + act_dim, 1, g) for _ in range(2)]
    for i, w in enumerate(ws):
        mlp.set_weights(i, *w)
    obs = torch.randn(M, obs_dim, device="cuda", generator=g)
    act = torch.tanh(torch.randn(M, act_dim, device="cuda", generator=g))
    q_full, q = _guarded((2, M, 1))
    da_full, da = _guarded((2, M, 16))
    rc = fwd_ex(mlp.h, obs.data_ptr(), obs_dim, act.data_ptr(), M, 2, 0, None, q_full.data_ptr(), None, None, None, da_full.data_ptr(), None, mlp._stream())
    assert rc == 0
    torch.cuda.synchronize()
    _check_guard(q_full, (2, M, 1))
    _check_guard(da_full, (2, M, 16))
    assert bool((da[:, :, act_dim:] == 0).all()), "columns beyond the action are not exactly zero"
    x64 = torch.cat([obs, act], 1).double().requires_grad_(True)
    m = dict(da_mirror=0.0, da_exact=0.0)
    for i in range(2):
        net = [t.double() for t in ws[i]]
        mir = R.dq_da(net, x64.detach(), obs_dim, act_dim, bf16=True)
        (gx,) = torch.autograd.grad(R.mlp_forward(net, x64)["y"].sum(), [x64])
        d = da[i, :, :act_dim].double()
        m["da_mirror"] = max(m["da_mirror"], float((d - mir).norm() / mir.norm()))
        m["da_exact"] = max(m["da_exact"], float((d - gx[:, obs_dim:]).norm() / gx[:, obs_dim:].norm()))
    mlp.close()
    return m


@pytest.mark.parametrize("M", [1, 129, 8192])
@pytest.mark.parametrize("obs_dim,act_dim", DA_SHAPES)
def test_dq_da_vs_float64(obs_dim, act_dim, M):
    m = dqda_metrics(obs_dim, act_dim, M, 0)
    assert m["da_mirror"] < TOL_DA_MIRROR and m["da_exact"] < (TOL_DA_EXACT_M1 if M == 1 else TOL_DA_EXACT), m
