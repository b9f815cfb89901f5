"""PARL-surface agent (`MujocoAgent.predict / sample / restore / save`, ETGRL/model/mujoco_agent.py:20-65) on top of the
fused wgmma MLP kernel (csrc/b2q_mlp.cu).  Parameters are held as float32 torch tensors under the reference's
state-dict key names (`actor_model.{l1,l2,mean_linear,std_linear}.{weight,bias}`, `critic_model.l1..l6.*`, SURVEY App. A)
so the reference's `.pt` checkpoints load unchanged; the kernel consumes bf16 images repacked on the device.
"""
import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import _lib

PREDICT, SAMPLE, RAW = 0, 1, 2
LOG_SIG_MAX, LOG_SIG_MIN = 2.0, -20.0   # mujoco_model.py:21-22


class FusedMLP:
    """ctypes handle of one b2q_mlp object: in_dim(<=64) -> 256 -> 256 -> out_dim(<=32), `nets` weight sets."""

    def __init__(self, in_dim, out_dim, nets=1, device=0, borrowed=None):
        self._owned = borrowed is None
        if not torch.cuda.is_available():
            raise RuntimeError("FusedMLP needs a CUDA device (wgmma kernel, no fallback)")
        self.lib = _lib.load()
        self.in_dim, self.out_dim, self.nets = in_dim, out_dim, nets
        self.device = torch.device("cuda", int(device))
        if borrowed is not None:
            self.h = C.c_void_p(borrowed)
            return
        self.h = C.c_void_p()
        rc = self.lib.b2q_mlp_create(int(device), in_dim, out_dim, nets, C.byref(self.h))
        if rc != 0:
            raise RuntimeError("b2q_mlp_create failed (%d)" % rc)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_weights(self, net, w1, b1, w2, b2, w3, b3):
        ts = [t.detach().to(self.device, torch.float32).contiguous() for t in (w1, b1, w2, b2, w3, b3)]
        assert ts[0].shape == (256, self.in_dim) and ts[2].shape == (256, 256) and ts[4].shape == (self.out_dim, 256)
        rc = self.lib.b2q_mlp_set_weights(self.h, net, *[t.data_ptr() for t in ts], self._stream())
        if rc != 0:
            raise RuntimeError("b2q_mlp_set_weights: %s" % self.lib.b2q_mlp_last_error(self.h).decode())
        self._keep = ts

    def forward(self, in1, in2=None, mode=PREDICT, seed=0, eps=None, want_raw=False, want_logp=False):
        in1 = in1.contiguous()
        M, d1 = in1.shape
        A = self.out_dim if mode == RAW else self.out_dim // 2
        out = torch.empty(self.nets, M, A, device=self.device, dtype=torch.float32)
        logp = torch.empty(self.nets, M, device=self.device, dtype=torch.float32) if (want_logp or mode == SAMPLE) else None
        raw = torch.empty(self.nets, M, self.out_dim, device=self.device, dtype=torch.float32) if want_raw else None
        p = lambda t: None if t is None else t.data_ptr()
        if in2 is not None:
            in2 = in2.contiguous()
        if eps is not None:
            eps = eps.contiguous()
        rc = self.lib.b2q_mlp_forward(self.h, in1.data_ptr(), d1, p(in2), M, mode, C.c_uint64(seed), p(eps), out.data_ptr(), p(logp), p(raw), self._stream())
        if rc != 0:
            raise RuntimeError("b2q_mlp_forward: %s" % self.lib.b2q_mlp_last_error(self.h).decode())
        return out, logp, raw

    def launch_count(self):
        return int(self.lib.b2q_mlp_launch_count(self.h))

    def close(self):
        if getattr(self, "h", None):
            if self._owned:
                self.lib.b2q_mlp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _init_linear(out_f, in_f, gen):
    # torch.nn.Linear default init (kaiming_uniform(a=sqrt(5)) -> U(-1/sqrt(in), 1/sqrt(in)) for weight and bias)
    bound = 1.0 / np.sqrt(in_f)
    w = (torch.rand(out_f, in_f, generator=gen) * 2 - 1) * bound
    b = (torch.rand(out_f, generator=gen) * 2 - 1) * bound
    return w, b


class MujocoAgent:
    """Batched drop-in for the reference agent: numpy [obs_dim] in -> numpy [act_dim] out like the reference, or
    device tensors [M, obs_dim] -> [M, act_dim] for rollouts (zero host traffic)."""

    def __init__(self, obs_dim, act_dim=12, device=0, seed=0):
        self.obs_dim, self.act_dim = obs_dim, act_dim
        self.device = torch.device("cuda", int(device))
        g = torch.Generator().manual_seed(seed)
        sd = OrderedDict()
        for name, (o, i) in (("actor_model.l1", (256, obs_dim)), ("actor_model.l2", (256, 256)), ("actor_model.mean_linear", (act_dim, 256)),
                             ("actor_model.std_linear", (act_dim, 256)), ("critic_model.l1", (256, obs_dim + act_dim)), ("critic_model.l2", (256, 256)),
                             ("critic_model.l3", (1, 256)), ("critic_model.l4", (256, obs_dim + act_dim)), ("critic_model.l5", (256, 256)),
                             ("critic_model.l6", (1, 256))):
            w, b = _init_linear(o, i, g)
            sd[name + ".weight"], sd[name + ".bias"] = w.to(self.device), b.to(self.device)
        self.params = sd
        self.actor = FusedMLP(obs_dim, 2 * act_dim, nets=1, device=device)
        self.critic = FusedMLP(obs_dim + act_dim, 1, nets=2, device=device)
        self._sample_calls = 0
        self.sync_weights()

    # ---- checkpoint surface (PARL: agent.save -> torch.save(state_dict), agent.restore: mujoco_agent.py:61-65)
    def state_dict(self):
        return OrderedDict((k, v.detach().cpu()) for k, v in self.params.items())

    def load_state_dict(self, sd):
        for k in self.params:
            if k not in sd:
                raise KeyError("checkpoint is missing %s" % k)
            if tuple(sd[k].shape) != tuple(self.params[k].shape):
                raise ValueError("shape mismatch for %s: %s vs %s" % (k, tuple(sd[k].shape), tuple(self.params[k].shape)))
            self.params[k] = sd[k].to(self.device, torch.float32).contiguous()
        self.sync_weights()
        for L in getattr(self, "_learners", {}).values():      # learners hold their own device copy of the parameters: refresh it, or the
            L.push()                                            # next learn() would overwrite the restored weights with the stale copy

    def save(self, path):
        torch.save(self.state_dict(), path)

    def restore(self, path):
        self.load_state_dict(torch.load(path, map_location="cpu"))

    def sync_weights(self):
        p = self.params
        self.actor.set_weights(0, p["actor_model.l1.weight"], p["actor_model.l1.bias"], p["actor_model.l2.weight"], p["actor_model.l2.bias"],
                               torch.cat([p["actor_model.mean_linear.weight"], p["actor_model.std_linear.weight"]], 0),
                               torch.cat([p["actor_model.mean_linear.bias"], p["actor_model.std_linear.bias"]], 0))
        self.critic.set_weights(0, p["critic_model.l1.weight"], p["critic_model.l1.bias"], p["critic_model.l2.weight"], p["critic_model.l2.bias"],
                                p["critic_model.l3.weight"], p["critic_model.l3.bias"])
        self.critic.set_weights(1, p["critic_model.l4.weight"], p["critic_model.l4.bias"], p["critic_model.l5.weight"], p["critic_model.l5.bias"],
                                p["critic_model.l6.weight"], p["critic_model.l6.bias"])

    # ---- batched device API
    def predict_batch(self, obs):
        return self.actor.forward(obs, mode=PREDICT)[0][0]

    def sample_batch(self, obs, eps=None, seed=None):
        self._sample_calls += 1
        out, logp, _ = self.actor.forward(obs, mode=SAMPLE, eps=eps, seed=self._sample_calls if seed is None else seed)
        return out[0], logp[0]

    def q_values(self, obs, act):
        out, _, _ = self.critic.forward(obs, in2=act, mode=RAW)
        return out[0, :, 0], out[1, :, 0]

    # ---- reference call shapes (numpy, batch 1): mujoco_agent.py:29-41
    def _single(self, obs, mode, seed):
        """One observation through the fused MLP with pinned host buffers as kernel arguments (the kernel reads the 49 floats
        from and writes the 12 actions to host memory over PCIe): one launch + one stream sync, no copy launches."""
        if getattr(self, "_h1", None) is None:
            A = self.act_dim
            self._h1 = (torch.empty(1, self.obs_dim).pin_memory(), torch.empty(1, 1, A).pin_memory(), torch.empty(1, 1).pin_memory())
            self._h1np = (self._h1[0].numpy(), self._h1[1].numpy())
        hin, hout, hlogp = self._h1
        self._h1np[0][0, :] = np.asarray(obs, dtype=np.float32).reshape(-1)
        a = self.actor
        st = torch.cuda.current_stream(a.device)
        rc = a.lib.b2q_mlp_forward(a.h, hin.data_ptr(), self.obs_dim, None, 1, mode, C.c_uint64(seed), None, hout.data_ptr(),
                                   hlogp.data_ptr() if mode == SAMPLE else None, None, C.c_void_p(st.cuda_stream))
        if rc != 0:
            raise RuntimeError("b2q_mlp_forward: %s" % a.lib.b2q_mlp_last_error(a.h).decode())
        st.synchronize()
        return self._h1np[1][0, 0].copy()

    def predict(self, obs):
        return self._single(obs, PREDICT, 0)

    def sample(self, obs):
        self._sample_calls += 1
        return self._single(obs, SAMPLE, self._sample_calls)


ACTOR_KEYS = ("actor_model.l1", "actor_model.l2")
CRITIC_NETS = (("critic_model.l1", "critic_model.l2", "critic_model.l3"), ("critic_model.l4", "critic_model.l5", "critic_model.l6"))


def flatten_params(p):
    """state-dict tensors -> the learner's flat vectors: actor [W1|b1|W2|b2|W3|b3] (W3 = cat(mean_linear, std_linear)), twin critic [2][...]."""
    a = torch.cat([p["actor_model.l1.weight"].reshape(-1), p["actor_model.l1.bias"], p["actor_model.l2.weight"].reshape(-1), p["actor_model.l2.bias"],
                   p["actor_model.mean_linear.weight"].reshape(-1), p["actor_model.std_linear.weight"].reshape(-1),
                   p["actor_model.mean_linear.bias"], p["actor_model.std_linear.bias"]])
    c = torch.cat([torch.cat([p[k + ".weight"].reshape(-1) if j == 0 else p[k + ".bias"] for k in net for j in (0, 1)]) for net in CRITIC_NETS])
    return a.contiguous(), c.contiguous()


def unflatten_params(p, a, c, obs_dim, act_dim):
    """inverse of flatten_params, writing into the state dict `p` (shapes taken from it)."""
    def take(vec, off, shape):
        n = int(np.prod(shape))
        return vec[off:off + n].reshape(shape).clone(), off + n
    off = 0
    for k in ("actor_model.l1", "actor_model.l2"):
        p[k + ".weight"], off = take(a, off, p[k + ".weight"].shape)
        p[k + ".bias"], off = take(a, off, p[k + ".bias"].shape)
    p["actor_model.mean_linear.weight"], off = take(a, off, p["actor_model.mean_linear.weight"].shape)
    p["actor_model.std_linear.weight"], off = take(a, off, p["actor_model.std_linear.weight"].shape)
    p["actor_model.mean_linear.bias"], off = take(a, off, p["actor_model.mean_linear.bias"].shape)
    p["actor_model.std_linear.bias"], off = take(a, off, p["actor_model.std_linear.bias"].shape)
    off = 0
    for net in CRITIC_NETS:
        for k in net:
            p[k + ".weight"], off = take(c, off, p[k + ".weight"].shape)
            p[k + ".bias"], off = take(c, off, p[k + ".bias"].shape)


class SACLearner:
    """SAC.learn on the device (csrc/b2q_sac.cu): same hyper-parameters and update order as ETGRL/alg/sac.py:30-118.
    `world`>1: data-parallel learner, gradient buckets all-reduced (NCCL) between the gradient and optimiser phases."""

    def __init__(self, agent, batch, gamma=0.99, tau=0.005, alpha=0.2, actor_lr=3e-4, critic_lr=3e-4, world=1, sync="exact", seed_key=0):
        """sync (world > 1): "exact" = the reference's update order (critic step, then the actor gradient against the UPDATED critic,
        sac.py:77-118) which needs two all-reduces; "flat" = both gradients against the pre-update parameters and ONE all-reduce of the
        single flat bucket [actor | critic] (SURVEY §8e).  sync="flat" with world == 1 runs the same phase order on one GPU.
        seed_key: added to the step seed of the phase-by-phase learn() (the path of world > 1), so data-parallel ranks draw different rsample() noise for
        their shards (train passes rank << 40: no step count reaches it); 0 keeps the single-GPU key."""
        self.lib = _lib.load()
        self.agent, self.batch, self.world, self.sync, self.seed_key = agent, batch, world, sync, int(seed_key)
        self.allreduce_events = None
        self.h = C.c_void_p()
        rc = self.lib.b2q_sac_create(agent.device.index or 0, agent.obs_dim, agent.act_dim, batch, gamma, tau, alpha, actor_lr, critic_lr, C.byref(self.h))
        if rc != 0:
            raise RuntimeError("b2q_sac_create failed (%d)" % rc)
        self.na, self.nc = self.lib.b2q_sac_param_count(self.h, 0), self.lib.b2q_sac_param_count(self.h, 1)
        # (critic_loss, actor_loss) of the last learn: a view of the learner's own accumulators (no copy node at the end of a learn); valid until the
        # next learn / bc_learn call starts
        self.losses = torch.as_tensor(_CudaBuf(self.lib.b2q_sac_loss_ptr(self.h), 2), device=agent.device)
        self.steps = 0
        self._graph = None
        self._static = None
        self._static_eps = [None, None]
        self.push()
        # forward objects that always see the parameters being trained (no weight copies during a rollout)
        self.actor = FusedMLP(agent.obs_dim, 2 * agent.act_dim, 1, agent.device.index or 0, borrowed=self.lib.b2q_sac_mlp(self.h, 0))
        self.critic = FusedMLP(agent.obs_dim + agent.act_dim, 1, 2, agent.device.index or 0, borrowed=self.lib.b2q_sac_mlp(self.h, 1))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.agent.device).cuda_stream)

    def push(self):
        a, c = flatten_params(self.agent.params)
        assert a.numel() == self.na and c.numel() == self.nc
        rc = self.lib.b2q_sac_set_params(self.h, a.data_ptr(), c.data_ptr(), None, self._stream())
        assert rc == 0
        self._keep = (a, c)

    def pull(self):
        a = torch.empty(self.na, device=self.agent.device); c = torch.empty(self.nc, device=self.agent.device)
        assert self.lib.b2q_sac_get_params(self.h, a.data_ptr(), c.data_ptr(), None, self._stream()) == 0
        unflatten_params(self.agent.params, a, c, self.agent.obs_dim, self.agent.act_dim)
        self.agent.sync_weights()

    def grads(self):
        a = torch.empty(self.na, device=self.agent.device); c = torch.empty(self.nc, device=self.agent.device)
        assert self.lib.b2q_sac_get_grads(self.h, a.data_ptr(), c.data_ptr(), self._stream()) == 0
        return a, c

    def _grad_view(self, which, n):
        # wrap the device bucket without copying (for in-place NCCL all-reduce)
        return torch.as_tensor(_CudaBuf(self.lib.b2q_sac_grad_ptr(self.h, which), n), device=self.agent.device)

    def _snapshot(self):
        """b2q_sac_snapshot_save into a new device byte tensor."""
        blob = torch.empty(int(self.lib.b2q_sac_snapshot_bytes(self.h)), dtype=torch.uint8, device=self.agent.device)
        rc = self.lib.b2q_sac_snapshot_save(self.h, blob.data_ptr(), self._stream())
        if rc != 0:
            raise RuntimeError("b2q_sac_snapshot_save: %d %s" % (rc, self.lib.b2q_sac_last_error(self.h).decode()))
        return blob

    def state_dict(self):
        """The learner's whole training state as CPU tensors: b2q_sac_snapshot_save (parameters, target, Adam moments, loss buffer, device
        step counter) and the host step count, which seeds the eager learn() and a captured one."""
        return {"snapshot": self._snapshot().cpu(), "steps": self.steps}

    def replica_state(self):
        """The part of the learner that data-parallel ranks keep identical, as one device byte tensor: the snapshot (parameters, target,
        Adam moments, device step counter) with its loss buffer, which holds this rank's shard losses, zeroed."""
        blob = self._snapshot()
        off = int(self.lib.b2q_sac_snapshot_loss_offset(self.h))
        blob[off:off + 4 * 4].zero_()                                   # the loss buffer: 4 floats
        return blob

    def load_state_dict(self, sd):
        """Restores a state_dict() of a learner with the same shapes and hyper-parameters, then pull()s the weights into the agent."""
        want = int(self.lib.b2q_sac_snapshot_bytes(self.h))
        blob = sd["snapshot"]
        if blob.dtype != torch.uint8 or blob.numel() != want:
            raise ValueError("learner snapshot of %d bytes, this learner's is %d" % (blob.numel() * blob.element_size(), want))
        blob = blob.to(self.agent.device)
        rc = self.lib.b2q_sac_snapshot_load(self.h, blob.data_ptr(), self._stream())
        if rc != 0:
            raise RuntimeError("b2q_sac_snapshot_load: %d %s" % (rc, self.lib.b2q_sac_last_error(self.h).decode()))
        self.steps = int(sd["steps"])
        self.pull()
        torch.cuda.current_stream(self.agent.device).synchronize()     # `blob` is freed on return

    def static_batch(self):
        """The learner's static input tensors (obs, act, rew, next_obs, term) of the CUDA-graph path.  Fill them in place (e.g.
        ReplayMemory.sample_batch(n, out=learner.static_batch())) and pass them to learn(graph=True): no per-step input copies."""
        if self._static is None:
            dev, B, D, A = self.agent.device, self.batch, self.agent.obs_dim, self.agent.act_dim
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
            self._static = [z(B, D), z(B, A), z(B), z(B, D), z(B)]
        return tuple(self._static[:5])

    def learn(self, obs, act, rew, next_obs, term, eps_next=None, eps_cur=None, pull=True, graph=False):
        """SAC.learn (alg/sac.py:77-118).  eps_next / eps_cur: the N(0,1) draws of the two rsample() calls; None (the production path) = drawn
        inside the kernels from a counter RNG keyed by (step seed, the learner's device-side step counter) — no noise tensors, and a CUDA-graph
        replay still draws fresh noise every step."""
        dev = self.agent.device
        t = lambda x: torch.as_tensor(x, dtype=torch.float32, device=dev).contiguous()
        obs, act, rew, next_obs, term = t(obs), t(act), t(rew).reshape(-1), t(next_obs), t(term).reshape(-1)
        assert obs.shape[0] == self.batch
        eps_next = None if eps_next is None else t(eps_next)
        eps_cur = None if eps_cur is None else t(eps_cur)
        pe = lambda x: None if x is None else x.data_ptr()
        self.steps += 1
        args = (obs.data_ptr(), act.data_ptr(), rew.data_ptr(), next_obs.data_ptr(), term.data_ptr(), pe(eps_next), pe(eps_cur), C.c_uint64(self.steps + self.seed_key))
        if self.world == 1 and graph:
            # one learner step replayed from a CUDA graph (static input buffers; inputs that already ARE the static buffers are not copied)
            ins = [obs, act, rew, next_obs, term]
            if self._graph is None:
                self.static_batch()
                self._static_eps = [None if e is None else torch.empty_like(e) for e in (eps_next, eps_cur)]
                sargs = tuple(x.data_ptr() for x in self._static[:5]) + tuple(pe(e) for e in self._static_eps) + (C.c_uint64(0),)
                for x, sx in zip(ins + [eps_next, eps_cur], self._static[:5] + self._static_eps):
                    if x is not None and x.data_ptr() != sx.data_ptr():
                        sx.copy_(x)
                side = torch.cuda.Stream(device=dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                self._graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self._graph, stream=side):
                    rc = self.lib.b2q_sac_learn(self.h, *sargs, None, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
                    assert rc == 0, rc
            if (eps_next is None) != (self._static_eps[0] is None) or (eps_cur is None) != (self._static_eps[1] is None):
                raise ValueError("learn(graph=True): explicit eps must be given either on every call or on none (the graph was captured with the other choice)")
            for x, sx in zip(ins + [eps_next, eps_cur], self._static[:5] + self._static_eps):
                if x is not None and x.data_ptr() != sx.data_ptr():
                    sx.copy_(x)
            self._graph.replay()
        elif self.sync == "flat":
            import torch.distributed as dist
            for ph in (0, 2):
                rc = self.lib.b2q_sac_phase(self.h, ph, *args, self._stream())
                if rc != 0:
                    raise RuntimeError("b2q_sac_phase %d: %d" % (ph, rc))
            if self.world > 1:
                g = self._grad_view(2, self.na + self.nc)
                if self.allreduce_events is not None:
                    self.allreduce_events[0].record()
                dist.all_reduce(g, op=dist.ReduceOp.AVG)          # ONE collective: 248 602 floats at obs 49 (NCCL averages in the reduction)
                if self.allreduce_events is not None:
                    self.allreduce_events[1].record()
            for ph in (1, 3):
                rc = self.lib.b2q_sac_phase(self.h, ph, *args, self._stream())
                if rc != 0:
                    raise RuntimeError("b2q_sac_phase %d: %d" % (ph, rc))
        elif self.world == 1:
            rc = self.lib.b2q_sac_learn(self.h, *args, None, self._stream())
            if rc != 0:
                raise RuntimeError("b2q_sac_learn: %d %s" % (rc, self.lib.b2q_sac_last_error(self.h).decode()))
        else:
            import torch.distributed as dist
            for ph in range(4):
                rc = self.lib.b2q_sac_phase(self.h, ph, *args, self._stream())
                if rc != 0:
                    raise RuntimeError("b2q_sac_phase %d: %d" % (ph, rc))
                if ph in (0, 2):   # one flat bucket per optimiser: all-reduce(mean) then the fused Adam kernel consumes it
                    g = self._grad_view(0 if ph == 2 else 1, self.na if ph == 2 else self.nc)
                    dist.all_reduce(g, op=dist.ReduceOp.AVG)
        if pull:
            self.pull()
        return self.losses

    def bc_learn(self, obs, ref_obs, ref_agent, eps=None, pull=True):
        """MujocoAgent.BClearn(obs, ref_obs, ref_agent) -> (critic_loss, actor_loss): mujoco_agent.py:56-60, alg/BC.py:53-72."""
        dev = self.agent.device
        t = lambda x: torch.as_tensor(x, dtype=torch.float32, device=dev).contiguous()
        obs, ref_obs = t(obs), t(ref_obs)
        eps = torch.randn(self.batch, self.agent.act_dim, device=dev) if eps is None else t(eps)
        rc = self.lib.b2q_sac_bc_learn(self.h, obs.data_ptr(), ref_obs.data_ptr(), ref_obs.shape[1], ref_agent.actor.h, ref_agent.critic.h, eps.data_ptr(),
                                       None, self._stream())
        if rc != 0:
            raise RuntimeError("b2q_sac_bc_learn: %d" % rc)
        if pull:
            self.pull()
        return self.losses

    def _bc_step(self, memory, expert, seed, acc):
        """gather the next batch on the device cursor, one seeded BC update (counter-RNG noise), add its losses to acc."""
        memory.gather_cursor(self._bc_perm, self._bc_cursor, self._bc_obs, self._bc_ref)
        rc = self.lib.b2q_sac_bc_learn_seeded(self.h, self._bc_obs.data_ptr(), self._bc_ref.data_ptr(), self._bc_ref.shape[1], expert.actor.h,
                                              expert.critic.h, None, C.c_uint64(seed), None, self._stream())
        if rc != 0:
            raise RuntimeError("b2q_sac_bc_learn_seeded: %d" % rc)
        acc.add_(self.losses)

    def bc_sweep(self, memory, expert, perm, n_batches, seed=0, graph_steps=64, pull=True):
        """n_batches BC updates (BCtrain.py:132-136) on the batches perm[k B:(k + 1) B], k = 0 .. n_batches - 1, of `memory` (a
        bc.BCReplayMemory), each one (device gather, b2q_sac_bc_learn_seeded with counter-RNG noise).  graph_steps G of them are captured
        once into one CUDA graph and replayed n_batches // G times; the n_batches % G left over run eagerly, so no batch is added or
        dropped.  No per-step host work, no per-step parameter pull: `pull` pulls once at the end.  Returns the device tensor [2] of the
        mean (critic_loss, actor_loss) over the updates."""
        dev, B = self.agent.device, self.batch
        if getattr(self, "_bc_perm", None) is None or self._bc_perm.numel() < memory.max_size or self._bc_ref.shape[1] != memory.ref_obs.shape[1]:
            self._bc_perm = torch.zeros(memory.max_size, dtype=torch.int64, device=dev)
            self._bc_cursor = torch.zeros(1, dtype=torch.int64, device=dev)
            self._bc_obs = torch.zeros(B, memory.obs.shape[1], device=dev)
            self._bc_ref = torch.zeros(B, memory.ref_obs.shape[1], device=dev)
            self._bc_acc = torch.zeros(2, device=dev)
            self._bc_graphs = {}
        assert perm.numel() >= n_batches * B
        self._bc_perm[:perm.numel()].copy_(perm)
        self._bc_cursor.zero_()
        self._bc_acc.zero_()
        G = max(1, int(graph_steps))
        if n_batches >= G:
            # the graph freezes every pointer it was captured with: key it by them
            key = (G, memory.obs.data_ptr(), memory.ref_obs.data_ptr(), int(expert.actor.h.value), int(expert.critic.h.value), int(seed))
            g = self._bc_graphs.get(key)
            if g is None:
                side = torch.cuda.Stream(device=dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    for _ in range(G):
                        self._bc_step(memory, expert, seed, self._bc_acc)
                self._bc_graphs[key] = g
            for _ in range(n_batches // G):
                g.replay()
        for _ in range(n_batches % G):
            self._bc_step(memory, expert, seed, self._bc_acc)
        if pull:
            self.pull()
        return self._bc_acc / max(n_batches, 1)

    def close(self):
        if getattr(self, "h", None):
            self.losses = self.losses.clone()      # the view of the learner's accumulators dies with the handle
            self._graph = None
            self._static = None
            self._bc_graphs = None
            self.lib.b2q_sac_destroy(self.h)
            self.h = None


class _CudaBuf:
    """Minimal __cuda_array_interface__ wrapper of a raw device float32 buffer (zero-copy view for torch.as_tensor)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<f4", "data": (int(ptr), False), "version": 3}


def _get_learner(self, n, actor_lr=3e-4, critic_lr=3e-4):
    """One SACLearner per (batch, learning rates), shared by learn() and BClearn(); agent.params is the single source of truth — a
    learner that was not the last one used re-reads it before stepping, so mixing learn / BClearn / restore never forks the weights."""
    if not hasattr(self, "_learners"):
        self._learners, self._active = {}, None
    key = (int(n), float(actor_lr), float(critic_lr))
    L = self._learners.get(key)
    if L is None:
        L = self._learners[key] = SACLearner(self, n, actor_lr=actor_lr, critic_lr=critic_lr)      # pushes agent.params
    elif self._active is not L:
        L.push()
    self._active = L
    return L


def _agent_learn(self, obs, action, reward, next_obs, terminal):
    """MujocoAgent.learn(obs, act, reward, next_obs, terminal) -> (critic_loss, actor_loss), mujoco_agent.py:43-54."""
    n = np.asarray(obs).shape[0] if not isinstance(obs, torch.Tensor) else obs.shape[0]
    l = _get_learner(self, n).learn(obs, action, reward, next_obs, terminal)
    return float(l[0]), float(l[1])


MujocoAgent.learn = _agent_learn


def _agent_bclearn(self, obs, ref_obs, ref_agent, actor_lr=3e-4, critic_lr=3e-4):
    l = _get_learner(self, obs.shape[0], actor_lr, critic_lr).bc_learn(obs, ref_obs, ref_agent)
    return float(l[0]), float(l[1])


MujocoAgent.BClearn = _agent_bclearn
