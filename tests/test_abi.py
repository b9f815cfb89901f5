"""The C-ABI shared library loads on a CPU-only box and exports every symbol the headers in include/ declare."""
import ctypes as C
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    syms = []
    for h in sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        src = re.sub(r"/\*.*?\*/", "", open(h).read(), flags=re.S)
        syms += re.findall(r"\b(b2q_[a-z0-9_]+)\s*\(", src)
    return sorted(set(syms))


def test_library_builds_loads_and_exports_every_declared_symbol():
    from paddlerobotics_b200 import build, _lib
    build.build()
    lib = C.CDLL(_lib.lib_path())
    decl = _declared_symbols()
    assert len(decl) >= 15
    missing = [s for s in decl if not hasattr(lib, s)]
    assert not missing, missing
    # and the Python loader binds exactly the declared set
    bound = set(_lib.SYMBOLS)
    assert bound == set(decl), (bound ^ set(decl))
    assert b"sm_90a" in _lib.load().b2q_version()


def test_config_struct_mirror_matches_header_defaults():
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import B2QConfig
    c = B2QConfig()
    _lib.load().b2q_default_config(C.byref(c))
    assert (c.sim_dt, c.action_repeat, c.solver_iters) == (0.002, 13, 23)
    assert c.solver_iters == int(300 / c.action_repeat)
    assert (c.erp, c.warmstart, c.contact_margin, c.foot_radius) == (0.2, 0.85, 0.02, 0.02)
    assert (c.w_torso, c.w_feet, c.w_up, c.w_tau, c.w_badfoot, c.w_footcontact, c.reward_p, c.vel_d) == (1.5, 0.3, 0.6, 0.07, 0.1, 0.1, 5.0, 0.5)  # train.py:461-487
    assert c.etg_T == 0.5 and c.etg_sigma_sq == 0.04 and c.etg_amp == 0.2 and c.ring_depth == 4   # 4*13-2 = 50 substeps = 100 ms >= the 80 ms cap of param2dynamic_dict (train.py:114)
    assert c.action_filter == 0 and c.filter_highcut == 4.0          # train.py:502, action_filter.py:44
    assert c.clip_motor_commands == 0 and c.max_angle_change == 0.2  # a1.py:229,62
    assert (c.sensor_dis, c.sensor_contact, c.sensor_imu, c.sensor_motor, c.sensor_etg, c.obs_normal) == (1, 1, 1, 1, 1, 1)   # train.py:494-500,473
    assert list(c.noise_stdev) == [0.0] * 5 and c.stuck_termination == 0 and c.body_collisions == 0 and c.motor_mode == 0
    assert c.joint_limits == 0 and c.external_force == 0 and list(c.base_damping) == [0.0] * 4 and c.etg_foot_y_inset == 0.0 and c.knee_contacts == 0
    c.threads_per_block = 256
    h = C.c_void_p()
    assert _lib.load().b2q_create(C.byref(c), C.byref(h)) == -1 and b"threads_per_block" in _lib.load().b2q_last_error(None)
    c.threads_per_block = 0; c.sensor_imu = 3
    assert _lib.load().b2q_create(C.byref(c), C.byref(h)) == -1 and b"sensor_imu" in _lib.load().b2q_last_error(None)


def test_create_fails_loudly_without_gpu_or_with_bad_config():
    import torch
    from paddlerobotics_b200 import _lib
    from paddlerobotics_b200._config import B2QConfig
    lib = _lib.load()
    c = B2QConfig(); lib.b2q_default_config(C.byref(c))
    h = C.c_void_p()
    c.num_envs = 0
    assert lib.b2q_create(C.byref(c), C.byref(h)) == -1 and b"num_envs" in lib.b2q_last_error(None)
    c.num_envs = 4
    if not torch.cuda.is_available():
        rc = lib.b2q_create(C.byref(c), C.byref(h))
        assert rc == -2 and b"no CPU fallback" in lib.b2q_last_error(None)      # B2Q_ECUDA: no silent CPU path
        from paddlerobotics_b200.env import VecQuadrupedalEnv
        with pytest.raises(RuntimeError):
            VecQuadrupedalEnv(4)
