"""Behaviour cloning of a partial-observation student from the SAC expert — the batched counterpart of ETGRL/BCtrain.py
(SURVEY §8f-3).  The student sees `obs[3:]` (no base displacement; that slot is a velocity estimate on hardware,
EnvWrapper.py:75-76) with sensor noise on rpy / drpy / q / qd (BCtrain.py:53-59); the expert sees the full observation.

    obs2noise(obs)            one row, NumPy global RNG, same draw order as the reference (bit-identical for one seed)
    obs2noise_batch(obs, gen) [N,49] device tensor, torch generator (the per-step path of the batched loop)
    cal_agent_obs / cal_ref_obs, BCReplayMemory (device ring of (student obs, expert obs) pairs, BCreplay_buffer.py:21-84;
                              observe / iter_pass: the fused noise + append kernel and the shuffled pass on a device cursor)
    run_bc(...)               collect with the student, clone from the expert with MujocoAgent.BClearn (alg/BC.py:53-72)
"""
import ctypes as C

import numpy as np
import torch

# slices and sigma / normalisation of BCtrain.py:55-58 (the obs row is already divided by the sensor normalisers)
NOISE = ((7, 10, 6e-2 / 0.1), (10, 13, 1e-1 / 0.5), (13, 25, 1e-2 / 0.1), (25, 37, 0.5))


def obs2noise(obs):
    """BCtrain.py:53-59, one observation row.  Draw order: rpy(3), drpy(3), q(12), qd(12) from np.random.normal."""
    o = np.array(obs, dtype=np.float64, copy=True)
    o[7:10] += np.random.normal(0, 6e-2, size=3) / 0.1
    o[10:13] += np.random.normal(0, 1e-1, size=3) / 0.5
    o[13:25] += np.random.normal(0, 1e-2, size=12) / 0.1
    o[25:37] += np.random.normal(0, 0.5, size=12)
    return o


def obs2noise_batch(obs, generator=None):
    """The same noise model on a [N,49] device tensor (one launch per slice, torch generator)."""
    o = obs.clone()
    for lo, hi, sig in NOISE:
        o[:, lo:hi] += torch.randn(o.shape[0], hi - lo, device=o.device, dtype=o.dtype, generator=generator) * sig
    return o


def cal_agent_obs(obs, sensor_noise=True, generator=None):
    """BCtrain.py:77-81: noisy student observation without the base-displacement slot."""
    if isinstance(obs, torch.Tensor):
        o = obs2noise_batch(obs, generator) if sensor_noise else obs
        return o[:, 3:].contiguous()
    o = obs2noise(obs) if sensor_noise else np.asarray(obs)
    return o[3:]


def cal_ref_obs(obs):
    """BCtrain.py:83-84."""
    return obs


class BCReplayMemory:
    """(student obs, expert obs) pairs on the device (alg/BCreplay_buffer.py:21-84: append, size, sample_batch_by_index)."""

    def __init__(self, max_size, obs_dim, ref_obs_dim, device="cuda"):
        self.max_size, self._size, self._pos = int(max_size), 0, 0
        self.obs = torch.zeros(self.max_size, obs_dim, device=device)
        self.ref_obs = torch.zeros(self.max_size, ref_obs_dim, device=device)

    def size(self):
        return self._size

    def append(self, obs, ref_obs):
        n = obs.shape[0]
        idx = (torch.arange(n, device=self.obs.device) + self._pos) % self.max_size
        self.obs[idx] = obs
        self.ref_obs[idx] = ref_obs
        self._pos = (self._pos + n) % self.max_size
        self._size = min(self.max_size, self._size + n)

    def sample_batch_by_index(self, idx):
        return self.obs[idx], self.ref_obs[idx]

    def state_dict(self):
        """The ring's rows up to the fill level and its cursor (position, fill level), as CPU tensors: a part-filled ring is not copied
        whole."""
        n = self._size
        return {"max_size": self.max_size, "obs_dim": self.obs.shape[1], "ref_obs_dim": self.ref_obs.shape[1], "obs": self.obs[:n].cpu(),
                "ref_obs": self.ref_obs[:n].cpu(), "pos": self._pos, "size": n}

    def load_state_dict(self, sd):
        """Restores a state_dict() into this memory's buffers (same capacity and widths); rows past the fill level are zeroed."""
        have = (self.max_size, self.obs.shape[1], self.ref_obs.shape[1])
        if (sd["max_size"], sd["obs_dim"], sd["ref_obs_dim"]) != have:
            raise ValueError("BC replay memory state of shape %s, this memory is %s" % ((sd["max_size"], sd["obs_dim"], sd["ref_obs_dim"]), have))
        n = int(sd["size"])
        for k in ("obs", "ref_obs"):
            buf = getattr(self, k)
            buf[:n].copy_(sd[k])
            buf[n:].zero_()
        self._pos, self._size = int(sd["pos"]), n
        torch.cuda.current_stream(self.obs.device).synchronize()     # the CPU sources must not be freed before the copies ran

    # ---- device path (b2q_bc_observe / b2q_bc_gather_cursor, include/b2q_rpm.h): float32 CUDA storage
    def observe(self, obs, step, noise=True, append=True, seed=0):
        """One control step in one launch: the student rows obs[:, 3:] + the sensor noise of BCtrain.py:53-59 (Philox key (seed, step),
        counter (env row, expert column)), and with append=True the pairs (student row, obs row) at the ring's host cursor
        (BCtrain.py:120).  obs: [N, 49] float32 CUDA tensor.  Returns the [N, 46] student rows."""
        from . import _lib
        obs = obs.contiguous()
        n, d = obs.shape
        assert obs.dtype == torch.float32 and obs.is_cuda and d == self.ref_obs.shape[1] and self.obs.shape[1] == d - 3
        student = torch.empty(n, d - 3, device=obs.device, dtype=torch.float32)
        ring = (self.obs.data_ptr(), self.ref_obs.data_ptr()) if append else (None, None)
        rc = _lib.load().b2q_bc_observe(obs.data_ptr(), n, d, student.data_ptr(), *ring, self._pos, self.max_size, int(seed) & 0xFFFFFFFF,
                                        int(step) & 0xFFFFFFFF, int(bool(noise)), C.c_void_p(torch.cuda.current_stream(obs.device).cuda_stream))
        if rc != 0:
            raise RuntimeError("b2q_bc_observe failed (%d)" % rc)
        if append:
            self._pos = (self._pos + n) % self.max_size
            self._size = min(self.max_size, self._size + n)
        return student

    def gather_cursor(self, perm, cursor, out_obs, out_ref):
        """Batch rows perm[cursor[0] + r] into out_obs / out_ref, then cursor[0] += batch (device int64 cursor: graph-capturable)."""
        from . import _lib
        rc = _lib.load().b2q_bc_gather_cursor(self.obs.data_ptr(), self.ref_obs.data_ptr(), perm.data_ptr(), perm.numel(), cursor.data_ptr(),
                                              out_obs.data_ptr(), out_ref.data_ptr(), out_obs.shape[0], self.obs.shape[1], self.ref_obs.shape[1],
                                              C.c_void_p(torch.cuda.current_stream(self.obs.device).cuda_stream))
        if rc != 0:
            raise RuntimeError("b2q_bc_gather_cursor failed (%d)" % rc)

    def iter_pass(self, batch, size=None, generator=None):
        """One shuffled pass of BCtrain.py:129-135 over the first `size` rows (default: all): a fresh device permutation and the batches
        perm[j:j + batch] for j in range(0, size - batch, batch), gathered on the device cursor.  Yields (obs, ref_obs) static buffers
        that the next batch overwrites."""
        size = self._size if size is None else int(size)
        dev = self.obs.device
        perm = torch.randperm(size, device=dev, generator=generator)
        cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        out = (torch.empty(batch, self.obs.shape[1], device=dev), torch.empty(batch, self.ref_obs.shape[1], device=dev))
        for _ in pass_offsets(size, batch):
            self.gather_cursor(perm, cursor, *out)
            yield out


def pass_offsets(size, batch):
    """The batch offsets of one pass over `size` rows, BCtrain.py:132 (the last full batch is never taken, as in the reference)."""
    return range(0, size - batch, batch)


def run_bc(env, student, expert, etg_w, etg_b, iters, batch=1024, act_bound=0.3, warmup=0, train_every=1, sensor_noise=True, memory=200000, seed=0,
           log_every=0):
    """Batched BCtrain.run_train_episode: the STUDENT acts (agent.sample on its noisy partial observation, BCtrain.py:105),
    pairs go to the replay, and every `train_every` control steps one shuffled minibatch is cloned with BClearn.
    `env` is a VecQuadrupedalEnv(auto_reset=True); returns the list of (critic_loss, actor_loss)."""
    gen = torch.Generator(device=env.device).manual_seed(seed)
    rpm = BCReplayMemory(memory, 46, 49, device=env.device)
    obs = env.reset(etg_w, etg_b).clone()
    losses = []
    for it in range(iters):
        a_obs = cal_agent_obs(obs, sensor_noise, gen)
        if rpm.size() < warmup:
            act = torch.rand(env.num_envs, 12, device=env.device, generator=gen) * 2 - 1
        else:
            act = student.sample_batch(a_obs, seed=it + 1)[0]
        nobs, rew, done, info = env.step(act * act_bound)
        rpm.append(a_obs, cal_ref_obs(obs))
        obs.copy_(nobs)
        if rpm.size() >= max(batch, warmup) and it % train_every == 0:
            idx = torch.randint(0, rpm.size(), (batch,), device=env.device, generator=gen)
            l = student.BClearn(*rpm.sample_batch_by_index(idx), expert)
            losses.append(l)
            if log_every and it % log_every == 0:
                print({"iter": it, "critic_loss": float(l[0]), "actor_loss": float(l[1]), "mean_step_reward": float(rew.mean())}, flush=True)
    return losses
