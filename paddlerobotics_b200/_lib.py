"""ctypes loader of csrc/libb2q.so (the C ABI in include/b2q.h).  Fails loudly: there is no fallback path."""
import ctypes as C
import os

from ._config import B2QConfig

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libb2q.so")
_lib = None

# every symbol include/b2q.h declares: (name, restype, argtypes)
_vp, _i, _u8p = C.c_void_p, C.c_int, C.c_void_p
SYMBOLS = {
    "b2q_default_config": (None, [C.POINTER(B2QConfig)]),
    "b2q_create": (_i, [C.POINTER(B2QConfig), C.POINTER(_vp)]),
    "b2q_destroy": (_i, [_vp]),
    "b2q_last_error": (C.c_char_p, [_vp]),
    "b2q_version": (C.c_char_p, []),
    "b2q_num_envs": (_i, [_vp]),
    "b2q_obs_dim": (_i, [_vp]),
    "b2q_act_dim": (_i, [_vp]),
    "b2q_info_dim": (_i, [_vp]),
    "b2q_elem_size": (_i, [_vp]),
    "b2q_set_dynamics": (_i, [_vp, _u8p, _vp, _vp]),
    "b2q_reset": (_i, [_vp, _u8p, _vp, _vp, _vp, _vp]),
    "b2q_reset_ex": (_i, [_vp, _u8p, _vp, _vp, _vp, _vp, _vp]),
    "b2q_set_external_force": (_i, [_vp, _vp, _vp]),
    "b2q_step": (_i, [_vp, _vp, _i, _vp, _vp, _u8p, _vp, _vp]),
    "b2q_step_host": (_i, [_vp, _vp, _i, _vp, _vp, _u8p, _vp, _vp]),
    "b2q_host_alloc": (_vp, [C.c_size_t]),
    "b2q_host_free": (None, [_vp]),
    "b2q_get_state": (_i, [_vp, _vp, _vp]),
    "b2q_set_state": (_i, [_vp, _vp, _vp]),
    "b2q_get_step_count": (_i, [_vp, _vp, _vp]),
    "b2q_launch_count": (C.c_int64, [_vp]),
    "b2q_set_max_episode_steps": (_i, [_vp, _i]),
    "b2q_snapshot_bytes": (C.c_int64, [_vp]),
    "b2q_snapshot_save": (_i, [_vp, _vp, _vp]),
    "b2q_snapshot_load": (_i, [_vp, _vp, _vp]),
    "b2q_set_terrain_tiles": (_i, [_vp, _vp, _i, _vp, _vp]),
    # policy / critic MLP forward on wgmma tensor cores — include/b2q_mlp.h
    "b2q_mlp_create": (_i, [_i, _i, _i, _i, C.POINTER(_vp)]),
    "b2q_mlp_destroy": (_i, [_vp]),
    "b2q_mlp_last_error": (C.c_char_p, [_vp]),
    "b2q_mlp_set_weights": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2q_mlp_forward": (_i, [_vp, _vp, _i, _vp, _i, _i, C.c_uint64, _vp, _vp, _vp, _vp, _vp]),
    "b2q_mlp_launch_count": (C.c_int64, [_vp]),
    # SAC learner — include/b2q_sac.h
    "b2q_sac_create": (_i, [_i, _i, _i, _i, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.POINTER(_vp)]),
    "b2q_sac_destroy": (_i, [_vp]),
    "b2q_sac_last_error": (C.c_char_p, [_vp]),
    "b2q_sac_param_count": (_i, [_vp, _i]),
    "b2q_sac_set_params": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "b2q_sac_get_params": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "b2q_sac_get_grads": (_i, [_vp, _vp, _vp, _vp]),
    "b2q_sac_learn": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint64, _vp, _vp]),
    "b2q_sac_phase": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint64, _vp]),
    "b2q_sac_bc_learn": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "b2q_sac_bc_learn_seeded": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, C.c_uint64, _vp, _vp]),
    "b2q_sac_mlp": (_vp, [_vp, _i]),
    "b2q_sac_grad_ptr": (_vp, [_vp, _i]),
    "b2q_sac_loss_ptr": (_vp, [_vp]),
    "b2q_sac_launch_count": (C.c_int64, [_vp]),
    "b2q_sac_snapshot_bytes": (C.c_int64, [_vp]),
    "b2q_sac_snapshot_loss_offset": (C.c_int64, [_vp]),
    "b2q_sac_snapshot_save": (_i, [_vp, _vp, _vp]),
    "b2q_sac_snapshot_load": (_i, [_vp, _vp, _vp]),
    # ES population fitness — include/b2q_es.h
    "b2q_es_accumulate": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b2q_es_accumulate_terms": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, C.c_double, _vp, _i, _i, _vp]),
    "b2q_train_episode_stats": (_i, [_vp, _vp, _vp, _i, _vp, _i, _i, C.c_double, _vp, _vp, _i, _i, _vp]),
    "b2q_es_fitness": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b2q_dyn_accumulate": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b2q_dyn_finish": (_i, [_vp, _i, _vp, _i, _i, _vp]),
    "b2q_etg_fit": (_i, [_vp, _vp, _vp, _vp, _vp, C.c_double, C.c_double, _vp, _vp, _i, _vp]),
    # device replay memory — include/b2q_rpm.h
    "b2q_rpm_append": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b2q_rpm_sample": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, C.c_uint64, _vp]),
    "b2q_rpm_append_cursor": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "b2q_rpm_sample_cursor": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, C.c_uint64, _vp, _vp]),
    "b2q_rpm_append_masked_cursor": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u8p, _i, _i, _i, _i, _vp, _vp]),
    "b2q_bc_observe": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _i, C.c_uint32, C.c_uint32, _i, _vp]),
    "b2q_bc_gather_cursor": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    # camera images — include/b2q_render.h
    "b2q_render": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    # deployment rehearsal — include/b2q_deploy.h
    "b2q_deploy_obs": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _vp]),
    "b2q_deploy_act": (_i, [_vp, _vp, C.c_double, _vp, _i, _vp, _vp, _i, _vp]),
    "b2q_bezier_reset": (_i, [_vp, _vp, _vp]),
    "b2q_bezier_act": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp]),
}


def lib_path():
    return _LIB_PATH


def load():
    """Returns the loaded library; raises if it was not built (run `python -m paddlerobotics_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            "paddlerobotics_b200: %s is missing — build it with `python -m paddlerobotics_b200.build` "
            "(nvcc, sm_90a). There is no CPU/PyTorch fallback for this path." % _LIB_PATH)
    lib = C.CDLL(_LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
