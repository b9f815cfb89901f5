"""bctrain (the batched BCtrain.py) without a device: its flag defaults against BCtrain.py:330-375 and :34-40, the options it refuses
before any device work, and the training schedule of run_train_episode (BCtrain.py:123-136)."""
import numpy as np
import pytest

# BCtrain.py:330-375 (flag defaults) and :34-40 (module constants that became batched flags)
REFERENCE_DEFAULTS = {
    "outdir": "BCtrain_log", "max_steps": 1e6, "load": "", "eval": 0, "suffix": "exp0", "task_mode": "stairstair", "step_y": 0.05,
    "random_dynamic": 0, "random_force": 0, "render": 0, "normal": 1, "vel_d": 0.6, "ETG": 1, "ETG_T": 0.5, "reward_p": 1, "e_step": 400,
    "act_mode": "traj", "ref_agent": "data/model/StairStair_3_itr_960231.pt", "ETG_path": "data/model/StairStair_3_itr_960231.npz",
    "ETG_H": 20, "stand": 0, "torso": 1, "up": 0.1, "tau": 0.1, "feet": 0.1, "act_bound": 0.3, "sensor_dis": 1, "sensor_motor": 1,
    "sensor_imu": 1, "sensor_contact": 1, "sensor_ETG": 1, "sensor_footpose": 0, "sensor_ETG_obs": 0, "sensor_dynamic": 0,
    "sensor_exforce": 0, "sensor_noise": 1, "RNN_mode": "None", "agent_mode": "None", "enable_action_filter": 0, "x_noise": 0,
    # WARMUP_STEPS, EVAL_EVERY_STEPS, MEMORY_SIZE, TRAIN_PER_STEPS, TRAIN_PER_TIME, BATCH_SIZE
    "warmup": 200, "eval_every_steps": 1e4, "memory": 1e7, "train_per_steps": 1024, "train_per_time": 10, "batch": 1024,
}


def test_flag_defaults_are_the_reference_values():
    from paddlerobotics_b200 import bctrain
    a = bctrain.parser().parse_args([])
    for k, v in REFERENCE_DEFAULTS.items():
        assert getattr(a, k) == v, (k, getattr(a, k), v)
    assert a.dynamic_param == ""                    # nominal dynamics: the reference's data file is not in its tree
    # act_bound per act_mode, BCtrain.py:238-243
    assert np.array_equal(bctrain.act_bound_of(a), [0.3] * 12)
    assert np.array_equal(bctrain.act_bound_of(bctrain.parser().parse_args(["--act_mode", "pose"])), [0.1, 0.7, 0.7] * 4)
    assert np.array_equal(bctrain.act_bound_of(bctrain.parser().parse_args(["--act_mode", "torque"])), [10] * 12)
    assert np.array_equal(bctrain.act_bound_of(bctrain.parser().parse_args(["--act_bound", "0.2"])), [0.2] * 12)


@pytest.mark.parametrize("flags", [["--agent_mode", "stack"], ["--RNN_mode", "GRU"], ["--sensor_footpose", "1"], ["--sensor_ETG_obs", "1"],
                                   ["--sensor_dynamic", "1"], ["--sensor_exforce", "1"], ["--random_dynamic", "1"], ["--stand", "0.5"],
                                   ["--render", "1"], ["--random_force", "1"], ["--sensor_imu", "2"], ["--x_noise", "1"]])
def test_unsupported_flags_raise_before_any_device_work(flags, monkeypatch):
    import torch
    from paddlerobotics_b200 import bctrain

    def no_device(*a, **k):
        raise AssertionError("device touched before the option check")
    monkeypatch.setattr(torch.cuda, "_lazy_init", no_device)
    monkeypatch.setattr(bctrain, "MujocoAgent", no_device)
    monkeypatch.setattr(bctrain, "make_vec_env", no_device)
    monkeypatch.setattr(bctrain, "etg_of_path", no_device)
    with pytest.raises(NotImplementedError):
        bctrain.main(flags)


def reference_batches(max_steps, tps, tpt, batch, memory, warmup):
    """BCtrain.py:123-136 counted per env step, at the step of each multiple of TRAIN_PER_STEPS: TRAIN_PER_TIME passes of
    range(0, size - BATCH, BATCH) over the ring's size then.  Returns the list of (multiple, size, offsets) per pass."""
    out = []
    for t in range(1, max_steps + 1):
        size = min(t, memory)
        if size >= warmup and t % tps == 0:
            out += [(t, size, list(range(0, size - batch, batch)))] * tpt
    return out


@pytest.mark.parametrize("n,tps,tpt,batch,memory,warmup,G", [
    (512, 1024, 10, 1024, 10 ** 7, 200, 64),          # BCtrain's constants, fewer envs than TRAIN_PER_STEPS
    (4096, 1024, 10, 1024, 10 ** 7, 200, 64),         # four multiples per control step
    (1000, 1024, 3, 256, 20000, 200, 7),              # multiples between control steps, a ring that fills up, partial graph chunks
    (300, 500, 2, 128, 3000, 1600, 5),                # warm-up larger than the first multiples
])
def test_sweep_schedule_is_the_reference_schedule(n, tps, tpt, batch, memory, warmup, G):
    from paddlerobotics_b200.bctrain import sweep_schedule
    steps = 60
    got = []
    for it in range(steps):
        for m, size, offsets, chunks in sweep_schedule(it * n, n, tps, tpt, batch, memory, warmup, G):
            assert it * n < m <= (it + 1) * n
            assert sum(chunks) == len(offsets) and all(0 < c <= G for c in chunks) and all(c == G for c in chunks[:-1])
            assert chunks == [G] * (len(offsets) // G) + ([len(offsets) % G] if len(offsets) % G else [])
            got.append((m, size, list(offsets)))
    ref = reference_batches(steps * n, tps, tpt, batch, memory, warmup)
    assert got == ref
    # the update count of the issue's estimate: 10 sum_k (k - 1) for multiples k * 1024 below the ring's capacity
    if (tps, tpt, batch, memory, warmup) == (1024, 10, 1024, 10 ** 7, 200):
        k_max = steps * n // 1024
        assert sum(len(o) for _, _, o in got) == 10 * sum(k - 1 for k in range(1, k_max + 1))


def test_pass_offsets_drop_the_last_full_batch_as_the_reference():
    from paddlerobotics_b200.bc import pass_offsets
    assert list(pass_offsets(1024, 1024)) == [] and list(pass_offsets(1025, 1024)) == [0] and list(pass_offsets(3072, 1024)) == [0, 1024]
    assert list(pass_offsets(100, 1024)) == []
