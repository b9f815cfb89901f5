"""Gym-style env surface of the reference (rlschool.make_env('Quadrupedal', ...): ETGRL/train.py:305-309) on top of
the CUDA engine.  Two classes:

* VecQuadrupedalEnv — N envs on one GPU.  Device API (torch tensors in/out, zero host traffic) for rollouts; host API
  (numpy in/out through pinned buffers) for callers that live on the CPU like the reference's train.py.
* QuadrupedalEnv    — N=1 wrapper with the reference's exact call shapes:
      obs, info = env.reset(ETG_w=w, ETG_b=b, x_noise=0)            (train.py:131)
      obs, reward, done, info = env.step(action, donef=False)         (train.py:147)
  `info` is a dict with the keys train.py consumes (velx, torso, feet, up, tau, ..., ETG_act, real_action,
  joint_angle, obs-IMU).

PyTorch is used only for device buffers / streams.  Every step runs in csrc/libb2q.so; nothing here computes physics.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._config import ACT_DIM, DYN_DIM, ETG_H, INFO, INFO_DIM, OBS_DIM, STATE_DIM, B2QConfig
from .etg import ETG_layer, Opt_with_points, dynamic_dict_to_row, param2dynamic_dict
from .terrain import TASKS, make_terrain

_CFG_KEYS = {f[0] for f in B2QConfig._fields_}


def _check(lib, h, rc, what):
    if rc != 0:
        msg = lib.b2q_last_error(h)
        raise RuntimeError("%s failed (%d): %s" % (what, rc, msg.decode() if msg else "?"))


class VecQuadrupedalEnv:
    def __init__(self, num_envs, device=0, precision="f32", auto_reset=False, heightfield=None, **cfg):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError("paddlerobotics_b200 needs a CUDA device: the hot path has no CPU fallback")
        self.device = torch.device("cuda", int(device))
        self.num_envs = int(num_envs)
        self.dtype = torch.float32 if precision in ("f32", 0) else torch.float64
        c = B2QConfig()
        self.lib.b2q_default_config(C.byref(c))
        c.num_envs, c.device, c.precision, c.auto_reset = self.num_envs, int(device), 0 if self.dtype == torch.float32 else 1, int(auto_reset)
        self._hf_keep = None
        self.n_tiles = 0            # > 0 once set_terrain_tiles made this a terrain-atlas env
        if heightfield is not None:
            hf, x0, y0, cell = heightfield
            hf = np.ascontiguousarray(hf, dtype=np.float64)
            self._hf_keep = hf
            c.terrain_type, c.hf_ny, c.hf_nx = 1, hf.shape[0], hf.shape[1]
            c.hf_x0, c.hf_y0, c.hf_cell = float(x0), float(y0), float(cell)
            c.hf_host = hf.ctypes.data_as(C.POINTER(C.c_double))
        for k, v in cfg.items():
            if k not in _CFG_KEYS:
                raise TypeError("unknown config key %r" % k)
            if k in ("noise_stdev", "base_damping"):
                arr = getattr(c, k)
                for i, x in enumerate(v):
                    arr[i] = float(x)
            else:
                setattr(c, k, v)
        self.cfg = c
        self.h = C.c_void_p()
        rc = self.lib.b2q_create(C.byref(c), C.byref(self.h))
        if rc != 0:
            raise RuntimeError("b2q_create failed (%d): %s" % (rc, self.lib.b2q_last_error(None).decode()))
        n, dev, dt = self.num_envs, self.device, self.dtype
        self.observation_dim = int(self.lib.b2q_obs_dim(self.h))          # <= 49: the sensor flags select blocks of the full layout
        self.action_dim = int(self.lib.b2q_act_dim(self.h))               # 12, or 60 in HYBRID mode (a 5-tuple per motor)
        self.obs = torch.zeros(n, self.observation_dim, device=dev, dtype=dt)
        self.reward = torch.zeros(n, device=dev, dtype=dt)
        self.done = torch.zeros(n, device=dev, dtype=torch.uint8)
        self.info = torch.zeros(n, INFO_DIM, device=dev, dtype=dt)
        self.control_dt = c.sim_dt * c.action_repeat
        # host API staging (pinned) — allocated lazily
        self._h_act = self._h_obs = self._h_rew = self._h_done = self._d_act = self._h_info = None

    # ------------------------------------------------------------------ device API
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _t(self, x, shape):
        t = torch.as_tensor(x, dtype=self.dtype, device=self.device)
        return t.expand(shape).contiguous() if tuple(t.shape) != tuple(shape) else t.contiguous()

    def set_dynamics(self, dyn=None, env_mask=None):
        """dyn: [N,48] rows (engine layout, see etg.dynamic_dict_to_row) or None for defaults; re-settles masked envs."""
        d = None if dyn is None else self._t(dyn, (self.num_envs, DYN_DIM))
        m = None if env_mask is None else torch.as_tensor(env_mask, dtype=torch.uint8, device=self.device).contiguous()
        _check(self.lib, self.h, self.lib.b2q_set_dynamics(self.h, None if m is None else m.data_ptr(), None if d is None else d.data_ptr(), self._stream()), "b2q_set_dynamics")

    def set_external_force(self, force=None):
        """World-frame push [N,3] applied at the base COM during every following step (None clears it); needs external_force=1."""
        f = None if force is None else self._t(force, (self.num_envs, 3))
        _check(self.lib, self.h, self.lib.b2q_set_external_force(self.h, None if f is None else f.data_ptr(), self._stream()), "b2q_set_external_force")

    def reset(self, ETG_w=None, ETG_b=None, env_mask=None, x_offset=None):
        """x_offset: [N] initial displacement of the base along x (what env.reset(x_noise=) randomises) or None."""
        w = None if ETG_w is None else self._t(torch.as_tensor(ETG_w, dtype=self.dtype).reshape(-1, 3, ETG_H), (self.num_envs, 3, ETG_H))
        b = None if ETG_b is None else self._t(torch.as_tensor(ETG_b, dtype=self.dtype).reshape(-1, 3), (self.num_envs, 3))
        m = None if env_mask is None else torch.as_tensor(env_mask, dtype=torch.uint8, device=self.device).contiguous()
        x = None if x_offset is None else self._t(x_offset, (self.num_envs,))
        p = lambda t: None if t is None else t.data_ptr()
        _check(self.lib, self.h, self.lib.b2q_reset_ex(self.h, p(m), p(w), p(b), p(x), self.obs.data_ptr(), self._stream()), "b2q_reset_ex")
        return self.obs

    def step(self, action, donef=False):
        """action: [N,12] device tensor (joint-space residual, already scaled by act_bound)."""
        a = action if (isinstance(action, torch.Tensor) and action.dtype == self.dtype and action.device == self.device and action.is_contiguous()) \
            else self._t(action, (self.num_envs, self.action_dim))
        rc = self.lib.b2q_step(self.h, a.data_ptr(), int(bool(donef)), self.obs.data_ptr(), self.reward.data_ptr(), self.done.data_ptr(),
                               self.info.data_ptr(), self._stream())
        if rc != 0:
            _check(self.lib, self.h, rc, "b2q_step")
        return self.obs, self.reward, self.done, self.info

    def get_state(self):
        s = torch.empty(self.num_envs, STATE_DIM, device=self.device, dtype=self.dtype)
        _check(self.lib, self.h, self.lib.b2q_get_state(self.h, s.data_ptr(), self._stream()), "b2q_get_state")
        return s

    def set_state(self, s):
        s = self._t(s, (self.num_envs, STATE_DIM))
        _check(self.lib, self.h, self.lib.b2q_set_state(self.h, s.data_ptr(), self._stream()), "b2q_set_state")

    def launch_count(self):
        return int(self.lib.b2q_launch_count(self.h))

    def set_max_episode_steps(self, m):
        """The per-env episode step limit of every following step (0 = none); episodes already running keep their step count."""
        _check(self.lib, self.h, self.lib.b2q_set_max_episode_steps(self.h, int(m)), "b2q_set_max_episode_steps")
        self.cfg.max_episode_steps = int(m)

    def set_terrain_tiles(self, tiles, tile_of_env):
        """Terrain atlas (b2q_set_terrain_tiles): env i reads the height field tiles[tile_of_env[i]] from now on.  tiles: [T, ny, nx] on this
        env's height-field grid (make_terrain_tiles gives such a stack), tile_of_env: [N] indices in [0, T).  Every env's reset snapshot is
        settled again on its tile with the dynamics it has; call reset() before the next step.  An atlas env has no state_dict,
        load_state_dict or get_camera_image."""
        if self.cfg.terrain_type != 1:
            raise ValueError("set_terrain_tiles needs an env built on a height field: the tiles share its grid")
        t = np.ascontiguousarray(tiles, dtype=np.float64)
        if t.ndim != 3 or t.shape[1:] != (self.cfg.hf_ny, self.cfg.hf_nx):
            raise ValueError("tiles of shape %s, this env's grid needs [T, %d, %d]" % (list(t.shape), self.cfg.hf_ny, self.cfg.hf_nx))
        m = np.ascontiguousarray(tile_of_env, dtype=np.int32).reshape(-1)
        if m.shape[0] != self.num_envs:
            raise ValueError("tile_of_env has %d entries for %d envs" % (m.shape[0], self.num_envs))
        _check(self.lib, self.h, self.lib.b2q_set_terrain_tiles(self.h, t.ctypes.data, int(t.shape[0]), m.ctypes.data, self._stream()), "b2q_set_terrain_tiles")
        self.n_tiles = int(t.shape[0])

    def _refuse_atlas(self, what):
        if self.n_tiles:
            raise RuntimeError("%s: not on a terrain-atlas env (set_terrain_tiles): the snapshot and the camera know one height field" % what)

    def state_dict(self):
        """Everything a later step or reset reads (b2q_snapshot_save: the device pool and the episode step limit), plus the last step's
        outputs, as CPU tensors."""
        self._refuse_atlas("state_dict")
        blob = torch.empty(int(self.lib.b2q_snapshot_bytes(self.h)), dtype=torch.uint8, device=self.device)
        _check(self.lib, self.h, self.lib.b2q_snapshot_save(self.h, blob.data_ptr(), self._stream()), "b2q_snapshot_save")
        return {"snapshot": blob.cpu(), "max_episode_steps": int(self.cfg.max_episode_steps), "obs": self.obs.cpu(), "reward": self.reward.cpu(),
                "done": self.done.cpu(), "info": self.info.cpu()}

    def load_state_dict(self, sd):
        """Restores a state_dict() of an env built with the same configuration; raises ValueError for a blob of another size and
        RuntimeError (naming the first differing field) for one of another configuration."""
        self._refuse_atlas("load_state_dict")
        want = int(self.lib.b2q_snapshot_bytes(self.h))
        blob = sd["snapshot"]
        if blob.dtype != torch.uint8 or blob.numel() != want:
            raise ValueError("env snapshot of %d bytes, this env's is %d" % (blob.numel() * blob.element_size(), want))
        blob = blob.to(self.device)
        _check(self.lib, self.h, self.lib.b2q_snapshot_load(self.h, blob.data_ptr(), self._stream()), "b2q_snapshot_load")
        self.cfg.max_episode_steps = int(sd["max_episode_steps"])
        for k in ("obs", "reward", "done", "info"):
            getattr(self, k).copy_(sd[k])
        torch.cuda.current_stream(self.device).synchronize()     # `blob` is freed on return

    def get_camera_image(self, width=640, height=480, env_ids=None, view=None, proj=None):
        """Ray-cast camera images of the current state (b2q_render, include/b2q_render.h): view v shows env env_ids[v] (default
        every env).  view / proj: [16] (one matrix for every view) or [V,16] column-major pybullet matrices; None = the follow
        camera of each env (render.follow_camera).  Returns device tensors (rgba [V,H,W,4] uint8, depth [V,H,W] float32 OpenGL
        depth-buffer values, seg [V,H,W] int32), which the next call with the same sizes overwrites: the buffers are reused, so the
        call can be captured in a CUDA graph (pass env_ids / view / proj as device tensors or None there)."""
        self._refuse_atlas("get_camera_image")
        from . import render
        dev, W, H = self.device, int(width), int(height)
        if env_ids is None:
            if getattr(self, "_r_all", None) is None:
                self._r_all = torch.arange(self.num_envs, dtype=torch.int32, device=dev)
            ids = self._r_all
        else:
            ids = torch.as_tensor(env_ids, device=dev).to(torch.int32).reshape(-1).contiguous()
        V = int(ids.shape[0])
        key = (V, H, W)
        if getattr(self, "_r_key", None) != key:
            self._r_key = key
            self._r_rgba = torch.empty(V, H, W, 4, dtype=torch.uint8, device=dev)
            self._r_depth = torch.empty(V, H, W, dtype=torch.float32, device=dev)
            self._r_seg = torch.empty(V, H, W, dtype=torch.int32, device=dev)
            self._r_view = torch.empty(V, 16, dtype=torch.float32, device=dev)
            self._r_proj = torch.empty(V, 16, dtype=torch.float32, device=dev)
            self._r_proj_hw = None
        if getattr(self, "_r_state", None) is None:
            self._r_state = torch.empty(self.num_envs, STATE_DIM, device=dev, dtype=self.dtype)
        _check(self.lib, self.h, self.lib.b2q_get_state(self.h, self._r_state.data_ptr(), self._stream()), "b2q_get_state")
        if view is None:
            render.follow_view_matrices(self._r_state.index_select(0, ids.clamp(0, self.num_envs - 1).long())[:, :3], self._r_view)
        else:
            self._r_view.copy_(torch.as_tensor(view, dtype=torch.float32, device=dev).reshape(-1, 16).expand(V, 16))
        if proj is None:
            if self._r_proj_hw != (H, W):     # the default projection depends on the aspect only: uploaded once per size
                self._r_proj.copy_(torch.tensor(render.follow_camera((0, 0, 0), W, H)[1], dtype=torch.float32, device=dev).expand(V, 16))
                self._r_proj_hw = (H, W)
        else:
            self._r_proj.copy_(torch.as_tensor(proj, dtype=torch.float32, device=dev).reshape(-1, 16).expand(V, 16))
            self._r_proj_hw = None
        rc = self.lib.b2q_render(self.h, self._r_state.data_ptr(), ids.data_ptr(), V, self._r_view.data_ptr(), self._r_proj.data_ptr(), W, H,
                                   self._r_rgba.data_ptr(), self._r_depth.data_ptr(), self._r_seg.data_ptr(), self._stream())
        _check(self.lib, self.h, rc, "b2q_render")
        return self._r_rgba, self._r_depth, self._r_seg

    # ------------------------------------------------------------------ host API (numpy in / numpy out)
    def _host_bufs(self):
        if self._h_act is None:
            n, npdt = self.num_envs, self.dtype
            self._h_act = torch.empty(n, self.action_dim, dtype=npdt).pin_memory()
            es = self.obs.element_size()
            od = self.observation_dim
            self._h_out = torch.empty(n * (od + 1) * es + n, dtype=torch.uint8).pin_memory()     # obs | rew | done contiguous: one D2H
            self._h_obs = self._h_out[: n * od * es].view(npdt).reshape(n, od)
            self._h_rew = self._h_out[n * od * es: n * (od + 1) * es].view(npdt)
            self._h_done = self._h_out[n * (od + 1) * es:]
            self._np_act, self._np_obs, self._np_rew, self._np_done = self._h_act.numpy(), self._h_obs.numpy(), self._h_rew.numpy(), self._h_done.numpy()
            self._h_ptrs = (self._h_act.data_ptr(), self._h_obs.data_ptr(), self._h_rew.data_ptr(), self._h_done.data_ptr())   # fixed for the env's lifetime

    def step_host(self, action_np, donef=False, info=False):
        """The reference-facing call with HOST buffers (numpy in / numpy out), one C call and one stream sync: the step kernel
        reads the actions from and stores obs / reward / done to pinned host memory (b2q_step_host).  info=True also returns
        the [N,56] info rows.  The returned arrays are views of the pinned buffers (overwritten by the next call)."""
        if self._h_act is None:
            self._host_bufs()
        np.copyto(self._np_act, np.asarray(action_np).reshape(self.num_envs, self.action_dim), casting="same_kind")
        if info and self._h_info is None:
            self._h_info = torch.empty(self.num_envs, INFO_DIM, dtype=self.dtype).pin_memory()
            self._np_info = self._h_info.numpy()
            self._h_info_ptr = self._h_info.data_ptr()
        pa, po, pr, pd = self._h_ptrs
        rc = self.lib.b2q_step_host(self.h, pa, 1 if donef else 0, po, pr, pd, self._h_info_ptr if info else None, self._stream())
        if rc != 0:
            _check(self.lib, self.h, rc, "b2q_step_host")
        if info:
            return self._np_obs, self._np_rew, self._np_done, self._np_info
        return self._np_obs, self._np_rew, self._np_done

    def h2d_bytes_per_step(self):
        return self.num_envs * self.action_dim * self.obs.element_size()

    def d2h_bytes_per_step(self, info=False):
        es = self.obs.element_size()
        return self.num_envs * (self.observation_dim * es + es + 1 + (INFO_DIM * es if info else 0))

    def close(self):
        if getattr(self, "h", None):
            self.lib.b2q_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Space:
    def __init__(self, n):
        self.shape = (n,)


def info_dict(row):
    """[INFO_DIM] row -> the reference's info dict keys."""
    row = np.asarray(row, dtype=np.float64)
    d = {k: float(row[v]) for k, v in INFO.items() if isinstance(v, int)}
    d["ETG_act"] = row[INFO["ETG_act"]].copy()
    d["real_action"] = row[INFO["real_action"]].copy()
    d["joint_angle"] = row[INFO["joint_angle"]].copy()
    d["obs-IMU"] = np.concatenate([row[INFO["rpy"]], row[INFO["drpy"]]])
    return d


# rlschool.quadrupedal.envs.env_builder.SENSOR_MODE / MonitorEnv.Random_Param_Dict keys ([EXT] SURVEY App. B.1) with the defaults
# ETGRL/train.py:494-503 passes
SENSOR_MODE = {"dis": 1, "motor": 1, "imu": 1, "contact": 1, "footpose": 0, "ETG": 1, "ETG_obs": 0, "dynamic_vec": 0, "force_vec": 0, "noise": 0}
Random_Param_Dict = {"random_dynamics": 0, "random_force": 0}
_UNSUPPORTED_SENSORS = ("footpose", "ETG_obs", "dynamic_vec", "force_vec")     # rlschool-only blocks whose layout is not in the reference tree
SENSOR_NOISE_STDDEV = (0.01, 0.05, 0.1, 0.01, 0.05)   # used when sensor_mode["noise"]=1: angle rad, velocity rad/s, torque Nm, rpy rad, rpy rate rad/s


def _motor_mode(m):
    """robot_config.MotorControlMode (enum, its value, or its name) -> engine motor_mode; deployment/robots/robot_config.py:24-40."""
    if m is None:
        return 0
    name = getattr(m, "name", None)
    val = getattr(m, "value", m)
    if name == "POSITION" or val in (1, "POSITION", "pose", "traj"):
        return 0
    if name == "TORQUE" or val in (2, "TORQUE", "torque"):
        return 1
    if name == "HYBRID" or val in (3, "HYBRID", "hybrid"):
        return 2
    raise NotImplementedError("motor_control_mode %r: POSITION, TORQUE and HYBRID are provided (PWM raises in the reference's motor model too, laikago_motor.py:126-128)" % (m,))


def quadrupedal_config(task="stairstair", motor_control_mode=None, sensor_mode=None, normal=1, reward_param=None, ETG=1, ETG_T=0.5, reward_p=5,
                       random_param=None, ETG_H=20, vel_d=0.5, step_y=0.05, enable_action_filter=0, seed=0, terrain_param=None):
    """The engine configuration of rlschool.make_env('Quadrupedal', ...) for any number of envs: (VecQuadrupedalEnv keywords including the
    terrain's `heightfield`, the random_param flags).  Raises NotImplementedError for every option the engine does not provide."""
    if ETG_H != ETG_H_CONST:
        raise NotImplementedError("ETG_H must be %d (the RBF layer width is fixed in the kernel)" % ETG_H_CONST)
    if task not in TASKS:
        raise NotImplementedError("task %r is not provided (have: %s)" % (task, ", ".join(TASKS)))
    sm = dict(SENSOR_MODE)
    if sensor_mode:
        unknown = set(sensor_mode) - set(SENSOR_MODE) - {"RNN"}
        if unknown:
            raise NotImplementedError("sensor_mode keys %s are not provided" % sorted(unknown))
        sm.update({k: v for k, v in sensor_mode.items() if k != "RNN"})
        rnn = sensor_mode.get("RNN")
        if rnn and rnn.get("mode", "None") not in ("None", None):
            raise NotImplementedError("sensor_mode['RNN'] mode %r: wrap the env with paddlerobotics_b200.obs_history.ObservationHistory instead" % (rnn.get("mode"),))
    for k in _UNSUPPORTED_SENSORS:
        if sm.get(k):
            raise NotImplementedError("sensor_mode[%r]: this rlschool-only observation block is not provided (its layout is not in the reference tree)" % k)
    rp = dict(Random_Param_Dict)
    if random_param:
        unknown = set(random_param) - set(Random_Param_Dict)
        if unknown:
            raise NotImplementedError("random_param keys %s are not provided" % sorted(unknown))
        rp.update(random_param)
    cfg = dict(etg_T=float(ETG_T), etg_T2=float(ETG_T), reward_p=float(reward_p), vel_d=float(vel_d), etg_enabled=int(bool(ETG)),
               action_filter=int(bool(enable_action_filter)), motor_mode=_motor_mode(motor_control_mode),
               sensor_dis=int(bool(sm["dis"])), sensor_contact=int(bool(sm["contact"])), sensor_imu=int(sm["imu"]), sensor_motor=int(sm["motor"]),
               sensor_etg=int(bool(sm["ETG"])), obs_normal=int(bool(normal)), external_force=int(bool(rp["random_force"])),
               stuck_termination=1, body_collisions=1, joint_limits=1, knee_contacts=1, noise_seed=int(seed))
    if sm["noise"]:
        cfg["noise_stdev"] = SENSOR_NOISE_STDDEV
    if task == "balancebeam":
        cfg["etg_foot_y_inset"] = float(step_y)
    for k_ref, k_cfg in (("torso", "w_torso"), ("feet", "w_feet"), ("up", "w_up"), ("tau", "w_tau"), ("stand", "w_stand"),
                         ("badfoot", "w_badfoot"), ("footcontact", "w_footcontact"), ("done", "w_done")):
        if reward_param and k_ref in reward_param:
            cfg[k_cfg] = float(reward_param[k_ref])
    if reward_param and float(reward_param.get("stand", 0)) != 0:
        raise NotImplementedError("reward_param['stand'] != 0: the stand term is not provided")
    cfg["heightfield"] = make_terrain(task, step_y=float(step_y), **dict(terrain_param or {}))
    return cfg, rp


def apply_dynamic_param(env, path):
    """A command's --dynamic_param: PATH.npy holds a 48-vector in [-1, 1] (a dynamic_param{epoch}.npy of dynamic_train) that goes through
    param2dynamic_dict to every env of `env`; an empty path keeps the nominal dynamics.  Returns env."""
    if path:
        env.set_dynamics(np.repeat(dynamic_param_row(path)[None], env.num_envs, 0))
    return env


def dynamic_param_row(path):
    """The [48] engine row of a command's --dynamic_param (see apply_dynamic_param): the nominal row when `path` is empty."""
    return dynamic_dict_to_row(param2dynamic_dict(np.load(path).reshape(-1))) if path else dynamic_dict_to_row()


def etg_of_path(ETG_path, ETG_T=0.5):
    """make_env's ETG_path rule: a `.npz` path gives its (w, b); anything else the default gait fit (train.py:298-299 defaults)."""
    if ETG_path not in (None, "None", "") and str(ETG_path).endswith(".npz"):
        z = np.load(ETG_path)
        return z["w"], z["b"]
    layer = ETG_layer(ETG_T, 0.026, ETG_H, 0.04, np.array([-np.pi / 2, 0]), 0.2, ETG_T)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=ETG_T, Footheight=0.1, Steplength=0.05)
    return w, b


class QuadrupedalEnv:
    """N=1 mirror of the reference env object (numpy in/out): rlschool.make_env('Quadrupedal', ...) of ETGRL/train.py:305-309.
    Every keyword of that call is honoured or raises NotImplementedError — nothing is swallowed."""

    def __init__(self, task="stairstair", motor_control_mode=None, render=False, sensor_mode=None, normal=1, dynamic_param=None,
                 reward_param=None, ETG=1, ETG_T=0.5, reward_p=5, ETG_path="None", random_param=None, ETG_H=20, vel_d=0.5,
                 step_y=0.05, enable_action_filter=0, device=0, precision="f32", seed=0, terrain_param=None, **engine_cfg):
        if render:
            raise NotImplementedError("render=True: there is no GUI / camera on the GPU path")
        cfg, rp = quadrupedal_config(task=task, motor_control_mode=motor_control_mode, sensor_mode=sensor_mode, normal=normal, reward_param=reward_param,
                                     ETG=ETG, ETG_T=ETG_T, reward_p=reward_p, random_param=random_param, ETG_H=ETG_H, vel_d=vel_d, step_y=step_y,
                                     enable_action_filter=enable_action_filter, seed=seed, terrain_param=terrain_param)
        self._random_dynamics, self._random_force = bool(rp["random_dynamics"]), bool(rp["random_force"])
        self._rng = np.random.default_rng(seed)
        hf = cfg.pop("heightfield")
        cfg.update(engine_cfg)
        self.task = task
        self.vec = VecQuadrupedalEnv(1, device=device, precision=precision, heightfield=hf, **cfg)
        self._dyn_row = dynamic_dict_to_row(dynamic_param) if dynamic_param else None
        if self._dyn_row is not None:
            self.vec.set_dynamics(self._dyn_row[None, :])
        self.observation_space, self.action_space = _Space(self.vec.observation_dim), _Space(self.vec.action_dim)
        self._w, self._b = etg_of_path(ETG_path, ETG_T)

    def reset(self, ETG_w=None, ETG_b=None, x_noise=0, hardset=None, dynamic_param=None):
        if hardset is not None:
            raise NotImplementedError("reset(hardset=...) is not provided")
        if dynamic_param is not None:
            self._dyn_row = dynamic_dict_to_row(dynamic_param)
            self.vec.set_dynamics(self._dyn_row[None, :])
        elif self._random_dynamics:     # random_param['random_dynamics'] (train.py:253): a fresh draw of the 48 dynamics parameters per episode
            self.vec.set_dynamics(dynamic_dict_to_row(param2dynamic_dict(self._rng.uniform(-1, 1, 48)))[None, :])
        if ETG_w is not None:
            self._w = np.asarray(ETG_w)
        if ETG_b is not None:
            self._b = np.asarray(ETG_b)
        # x_noise (train.py:131,505): the episode starts displaced along x so that the gait phase at the first obstacle varies
        xo = np.array([self._rng.uniform(-0.1, 0.1)]) if x_noise else None
        if self._random_force:          # random_param['random_force'] (train.py:254): a horizontal push, redrawn every episode
            ang, mag = self._rng.uniform(0, 2 * np.pi), self._rng.uniform(0, 15.0)
            self.vec.set_external_force(np.array([[mag * np.cos(ang), mag * np.sin(ang), 0.0]]))
        obs = self.vec.reset(self._w, self._b, x_offset=xo)
        info = {"ETG_act": np.zeros(12)}
        return obs[0].double().cpu().numpy(), info

    def step(self, action, donef=False):
        # one C call + one stream sync: actions in, obs / reward / done / info out through pinned host buffers
        obs, rew, done, info = self.vec.step_host(np.asarray(action).reshape(1, self.vec.action_dim), donef, info=True)
        return obs[0].astype(np.float64), float(rew[0]), bool(done[0]), info_dict(info[0])

    def get_camera_image(self, width=640, height=480, viewMatrix=None, projectionMatrix=None):
        """pybullet.getCameraImage(width, height, viewMatrix, projectionMatrix) -> (width, height, rgba [H,W,4] uint8,
        depth [H,W] float32, seg [H,W] int32) as numpy arrays (train.py:197).  No matrices = the follow camera."""
        rgba, depth, seg = self.vec.get_camera_image(width, height, view=viewMatrix, proj=projectionMatrix)
        return int(width), int(height), rgba[0].cpu().numpy(), depth[0].cpu().numpy(), seg[0].cpu().numpy()

    def close(self):
        self.vec.close()


ETG_H_CONST = ETG_H


def make_env(name, **kwargs):
    """rlschool.make_env('Quadrupedal', task=..., motor_control_mode=..., ...) — ETGRL/train.py:305-309."""
    if name != "Quadrupedal":
        raise NotImplementedError("only 'Quadrupedal' is provided")
    return QuadrupedalEnv(**kwargs)
