"""Device-resident replay memory (SURVEY §8f-2) with the call surface of parl.utils.ReplayMemory as the reference uses it
(`rpm.append(obs, action, reward, next_obs, terminal)`, `rpm.sample_batch(B)`, `rpm.size()`: ETGRL/train.py:159,164,142),
batched over envs: append() takes [N, ...] device tensors (one transition per env per control step)."""
import ctypes as C

import torch

from . import _lib


class ReplayMemory:
    def __init__(self, max_size, obs_dim, act_dim, device=0, device_cursor=False):
        """device_cursor=True keeps the ring position, the fill level and the sample counter in device memory (b2q_rpm_*_cursor): append /
        sample_batch then take nothing step-dependent as a kernel argument and can be captured in a CUDA graph.  The host-side mirrors
        (size()) advance identically."""
        self.lib = _lib.load()
        self.max_size, self.obs_dim, self.act_dim = int(max_size), obs_dim, act_dim
        self.device = torch.device("cuda", int(device))
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)
        self.obs, self.next_obs = z(self.max_size, obs_dim), z(self.max_size, obs_dim)
        self.action, self.reward, self.terminal = z(self.max_size, act_dim), z(self.max_size), z(self.max_size)
        self._curr_size, self._curr_pos, self._samples = 0, 0, 0
        self.cursor = torch.zeros(3, dtype=torch.int64, device=self.device) if device_cursor else None   # {position, fill level, samples}
        # append_masked: how many rows it wrote is known only on the device, so it runs on a device cursor (self.cursor, or in host-cursor
        # mode this one, loaded from the host mirrors) and leaves the mirrors stale until sync_host() reads that cursor back
        self._masked_cursor = None
        self._stale = False

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def sync_host(self):
        """Brings the host mirrors (size(), the host-cursor position) up to date after masked appends with one device-to-host read of
        the cursor.  In device-cursor mode it always reads (call it after replaying a CUDA graph that contains a masked append); in
        host-cursor mode only when a masked append ran since the last read.  size(), append, advance and sample_batch catch up by
        themselves after eager masked appends."""
        if self.cursor is not None:
            self._stale = True
        self._refresh()

    def _refresh(self):
        if self._stale:
            self._curr_pos, self._curr_size = (int(x) for x in (self.cursor if self.cursor is not None else self._masked_cursor)[:2].tolist())
            self._stale = False

    def size(self):
        self._refresh()
        return self._curr_size

    def __len__(self):
        return self.size()

    def state_dict(self):
        """The ring's rows up to the fill level, the device cursor [position, fill level, samples] (None in host-cursor mode) and the host
        mirrors, as CPU tensors."""
        self._refresh()
        n = self._curr_size
        return {"max_size": self.max_size, "obs_dim": self.obs_dim, "act_dim": self.act_dim, "obs": self.obs[:n].cpu(), "action": self.action[:n].cpu(),
                "reward": self.reward[:n].cpu(), "next_obs": self.next_obs[:n].cpu(), "terminal": self.terminal[:n].cpu(),
                "cursor": None if self.cursor is None else self.cursor.cpu(), "pos": self._curr_pos, "size": n, "samples": self._samples}

    def load_state_dict(self, sd):
        """Restores a state_dict() into this memory's buffers (same capacity, widths and cursor mode); rows past the fill level are zeroed."""
        if (sd["max_size"], sd["obs_dim"], sd["act_dim"]) != (self.max_size, self.obs_dim, self.act_dim):
            raise ValueError("replay memory state of shape %s, this memory is %s" % ((sd["max_size"], sd["obs_dim"], sd["act_dim"]), (self.max_size, self.obs_dim, self.act_dim)))
        if (sd["cursor"] is None) != (self.cursor is None):
            raise ValueError("replay memory state and this memory differ in cursor mode (device cursor: %s here)" % (self.cursor is not None))
        n = int(sd["size"])
        for k in ("obs", "action", "reward", "next_obs", "terminal"):
            buf = getattr(self, k)
            buf[:n].copy_(sd[k])
            buf[n:].zero_()
        if self.cursor is not None:
            self.cursor.copy_(sd["cursor"])
        self._curr_pos, self._curr_size, self._samples = int(sd["pos"]), n, int(sd["samples"])
        self._stale = False
        torch.cuda.current_stream(self.device).synchronize()     # the CPU sources must not be freed before the copies ran

    def append_masked(self, obs, act, reward, next_obs, terminal, mask):
        """Appends the rows i with mask[i] != 0, in row order (one row per env whose transition is kept, e.g. the envs still in their
        first episode).  The number of rows written never reaches the host (b2q_rpm_append_masked_cursor): no sync, and in device-cursor
        mode the call can be captured in a CUDA graph and replayed with new mask contents."""
        t = lambda x: torch.as_tensor(x, dtype=torch.float32, device=self.device).contiguous()
        obs, act, reward, next_obs, terminal = t(obs).reshape(-1, self.obs_dim), t(act).reshape(-1, self.act_dim), t(reward).reshape(-1), t(next_obs).reshape(-1, self.obs_dim), t(terminal).reshape(-1)
        mask = torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous().reshape(-1)
        n = obs.shape[0]
        if not (act.shape[0] == reward.shape[0] == next_obs.shape[0] == terminal.shape[0] == mask.shape[0] == n):
            raise ValueError("append_masked: obs, act, reward, next_obs, terminal and mask must have the same number of rows")
        cursor = self.cursor
        if cursor is None:
            if self._masked_cursor is None:
                self._masked_cursor = torch.zeros(3, dtype=torch.int64, device=self.device)
            cursor = self._masked_cursor
            if not self._stale:                  # the host mirrors hold the position: load them (fills, no sync)
                cursor[0], cursor[1], cursor[2] = self._curr_pos, self._curr_size, self._samples
        rc = self.lib.b2q_rpm_append_masked_cursor(self.obs.data_ptr(), self.action.data_ptr(), self.reward.data_ptr(), self.next_obs.data_ptr(), self.terminal.data_ptr(),
                                                   obs.data_ptr(), act.data_ptr(), reward.data_ptr(), next_obs.data_ptr(), terminal.data_ptr(), mask.data_ptr(),
                                                   n, self.obs_dim, self.act_dim, self.max_size, cursor.data_ptr(), self._stream())
        assert rc == 0, rc
        self._keep_masked = (obs, act, reward, next_obs, terminal, mask)      # inputs of a captured launch must outlive the capture
        self._stale = True

    def append(self, obs, act, reward, next_obs, terminal):
        self._refresh()
        t = lambda x: torch.as_tensor(x, dtype=torch.float32, device=self.device).contiguous()
        obs, act, reward, next_obs, terminal = t(obs).reshape(-1, self.obs_dim), t(act).reshape(-1, self.act_dim), t(reward).reshape(-1), t(next_obs).reshape(-1, self.obs_dim), t(terminal).reshape(-1)
        n = obs.shape[0]
        if self.cursor is not None:
            rc = self.lib.b2q_rpm_append_cursor(self.obs.data_ptr(), self.action.data_ptr(), self.reward.data_ptr(), self.next_obs.data_ptr(), self.terminal.data_ptr(),
                                                obs.data_ptr(), act.data_ptr(), reward.data_ptr(), next_obs.data_ptr(), terminal.data_ptr(),
                                                n, self.obs_dim, self.act_dim, self.max_size, self.cursor.data_ptr(), self._stream())
            assert rc == 0, rc
            self._keep = (obs, act, reward, next_obs, terminal)      # inputs of a captured launch must outlive the capture
            self._curr_pos = (self._curr_pos + n) % self.max_size
            self._curr_size = min(self._curr_size + n, self.max_size)
            return
        rc = self.lib.b2q_rpm_append(self.obs.data_ptr(), self.action.data_ptr(), self.reward.data_ptr(), self.next_obs.data_ptr(), self.terminal.data_ptr(),
                                     obs.data_ptr(), act.data_ptr(), reward.data_ptr(), next_obs.data_ptr(), terminal.data_ptr(), None,
                                     n, self.obs_dim, self.act_dim, self._curr_pos, self.max_size, self._stream())
        assert rc == 0, rc
        self._curr_pos = (self._curr_pos + n) % self.max_size
        self._curr_size = min(self._curr_size + n, self.max_size)

    def advance(self, n, samples=1):
        """Host-side mirrors only: a captured iteration (device cursor) was replayed — n rows appended, `samples` minibatches drawn."""
        self._refresh()
        self._curr_pos = (self._curr_pos + n) % self.max_size
        self._curr_size = min(self._curr_size + n, self.max_size)
        self._samples += samples

    def sample_batch(self, batch_size, seed=None, out=None):
        """Uniform sample (replay_memory.py sample_batch).  out = (obs, act, rew, next_obs, term) float32 device tensors to gather into
        (e.g. SACLearner.static_batch(): the learner's CUDA-graph inputs are then filled in place, with no copy in between)."""
        self._refresh()
        self._samples += 1
        if out is not None:
            obs, act, rew, nobs, term = out
            assert obs.shape == (batch_size, self.obs_dim) and act.shape == (batch_size, self.act_dim) and all(x.is_contiguous() and x.dtype == torch.float32 for x in out)
        else:
            z = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
            obs, nobs, act, rew, term = z(batch_size, self.obs_dim), z(batch_size, self.obs_dim), z(batch_size, self.act_dim), z(batch_size), z(batch_size)
        if self.cursor is not None:
            rc = self.lib.b2q_rpm_sample_cursor(self.obs.data_ptr(), self.action.data_ptr(), self.reward.data_ptr(), self.next_obs.data_ptr(), self.terminal.data_ptr(),
                                                obs.data_ptr(), act.data_ptr(), rew.data_ptr(), nobs.data_ptr(), term.data_ptr(), batch_size, self.obs_dim, self.act_dim,
                                                C.c_uint64(0 if seed is None else seed), self.cursor.data_ptr(), self._stream())
            assert rc == 0, rc
            return obs, act, rew, nobs, term
        rc = self.lib.b2q_rpm_sample(self.obs.data_ptr(), self.action.data_ptr(), self.reward.data_ptr(), self.next_obs.data_ptr(), self.terminal.data_ptr(),
                                     obs.data_ptr(), act.data_ptr(), rew.data_ptr(), nobs.data_ptr(), term.data_ptr(), batch_size, self.obs_dim, self.act_dim,
                                     self._curr_size, C.c_uint64(self._samples if seed is None else seed), self._stream())
        assert rc == 0, rc
        return obs, act, rew, nobs, term
