"""deploy_test (the batched deployment/test.py) without a device: its flag defaults against test.py:108-126, the observation width of every
sensor combination against test.py's get_obs_dim, the inputs it refuses before any device work, and the layout of the batch."""
import itertools
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUDENT = os.path.join(ROOT, "tests", "golden", "StairStair3_BC1_itr_500383.pt")
CPG = os.path.join(ROOT, "tests", "golden", "gait_action_list_CPG_stairstair7_12_3.npy")

# deployment/test.py:108-126
REFERENCE_DEFAULTS = {
    "suffix": "exp0", "ETG_path": "exp/stair_6_21/gait_action_list_ETG_stair.npy", "sensor_dis": 0, "sensor_motor": 1, "sensor_imu": 1,
    "sensor_contact": 1, "sensor_footpose": 0, "sensor_ETG": 1, "timesteps": 5, "timeinterval": 1, "RNN_mode": "None", "dt": 0.026,
    "max_time": 1, "normal": 1, "gait": 0, "load": "", "enable_action_filter": 0,
}


def reference_get_obs_dim(sensor_mode):
    """test.py:26-46."""
    obs_dim = 0
    if "motor" in sensor_mode:
        if sensor_mode["motor"] == 1:
            obs_dim += 24
        elif sensor_mode["motor"] == 2:
            obs_dim += 12
    if "dis" in sensor_mode and sensor_mode["dis"]:
        obs_dim += 3
    if "imu" in sensor_mode:
        if sensor_mode["imu"] == 1:
            obs_dim += 6
        elif sensor_mode["imu"] == 2:
            obs_dim += 3
    if "contact" in sensor_mode and sensor_mode["contact"]:
        obs_dim += 4
    if "ETG" in sensor_mode and sensor_mode["ETG"]:
        obs_dim += 12
    rnn = sensor_mode.get("RNN")
    if rnn and rnn["time_steps"] > 0 and rnn["mode"] == "stack":
        obs_dim *= rnn["time_steps"] + 1
    return obs_dim


def test_flag_defaults_are_the_reference_values():
    from paddlerobotics_b200 import deploy_test
    a = deploy_test.parser().parse_args([])
    for k, v in REFERENCE_DEFAULTS.items():
        assert getattr(a, k) == v, (k, getattr(a, k), v)
    assert a.task_mode == "stairstair" and a.dynamic_param == [] and a.x_starts == 1
    assert deploy_test.steps_of(a) == 100


def test_obs_width_of_every_sensor_combination():
    """obs_dim_of equals get_obs_dim for every flag combination, and deploy_config selects that width with the ETG block last."""
    from paddlerobotics_b200 import deploy, deploy_test
    for dis, motor, imu, contact, etg in itertools.product((0, 1), (0, 1, 2), (0, 1, 2), (0, 1), (0, 1)):
        ref = reference_get_obs_dim({"dis": dis, "motor": motor, "imu": imu, "contact": contact, "ETG": etg,
                                     "RNN": {"time_steps": 5, "time_interval": 1, "mode": "None"}})
        assert deploy.obs_dim_of(dis, motor, imu, contact, etg) == ref
        if ref == 0:
            continue
        a = deploy_test.parser().parse_args(["--sensor_dis", str(dis), "--sensor_motor", str(motor), "--sensor_imu", str(imu),
                                             "--sensor_contact", str(contact), "--sensor_ETG", str(etg)])
        cfg = deploy.deploy_config(a)
        assert cfg["etg_enabled"] == 0 and cfg["sensor_etg"] == etg and cfg["obs_normal"] == 1
        assert (cfg["sensor_dis"], cfg["sensor_motor"], cfg["sensor_imu"], cfg["sensor_contact"]) == (dis, motor, imu, contact)

        class _Env:     # etg_col_of reads only these two attributes
            observation_dim = ref

            class cfg:
                sensor_etg = etg
        assert deploy.etg_col_of(_Env) == (ref - 12 if etg else -1)


def test_deploy_config_is_the_training_configuration_with_etg_off():
    from paddlerobotics_b200 import deploy, deploy_test
    cfg = deploy.deploy_config(deploy_test.parser().parse_args([]))
    assert (cfg["joint_limits"], cfg["knee_contacts"], cfg["stuck_termination"], cfg["body_collisions"]) == (1, 1, 1, 1)
    assert cfg["etg_enabled"] == 0 and cfg["action_filter"] == 0 and "noise_stdev" not in cfg
    assert cfg["heightfield"] is not None
    assert deploy.deploy_config(deploy_test.parser().parse_args(["--enable_action_filter", "1"]))["action_filter"] == 1


def _refused(tmp_path, flags, monkeypatch, exc, words):
    import torch
    from paddlerobotics_b200 import deploy_test

    def no_device(*a, **k):
        raise AssertionError("device touched before the input check")
    monkeypatch.setattr(torch.cuda, "_lazy_init", no_device)
    monkeypatch.setattr(deploy_test, "VecQuadrupedalEnv", no_device)
    monkeypatch.setattr(deploy_test, "rehearse", no_device)
    with pytest.raises(exc) as e:
        deploy_test.main(flags)
    for w in words:
        assert w in str(e.value), (w, str(e.value))


def test_refused_inputs_raise_before_any_device_work(tmp_path, monkeypatch):
    ok = ["--load", STUDENT, "--ETG_path", CPG]
    short = str(tmp_path / "short.npy"); np.save(short, np.zeros((100, 12)))
    wide = str(tmp_path / "wide.npy"); np.save(wide, np.zeros((200, 13)))
    flat = str(tmp_path / "flat.npy"); np.save(flat, np.zeros(1200))
    bad_dyn = str(tmp_path / "dyn.npy"); np.save(bad_dyn, np.zeros(47))
    for flags, exc, words in (
            (["--gait", "1"], NotImplementedError, ["--gait"]),
            (["--RNN_mode", "stack"], NotImplementedError, ["--RNN_mode", "--timesteps"]),
            (["--RNN_mode", "GRU", "--timesteps", "3"], NotImplementedError, ["--RNN_mode"]),
            (["--dt", "0.02"], ValueError, ["--dt"]),
            (["--ETG_path", short], ValueError, ["--ETG_path", "100 rows", "row 100"]),
            (["--ETG_path", CPG, "--max_time", "8"], ValueError, ["--ETG_path", "800 rows", "row 800"]),
            (["--ETG_path", wide], ValueError, ["--ETG_path", "[rows, 12]"]),
            (["--ETG_path", flat], ValueError, ["--ETG_path", "[rows, 12]"]),
            (["--sensor_dis", "1"], ValueError, ["--load", "46 inputs", "49-wide"]),
            (["--sensor_ETG", "0"], ValueError, ["--load", "46 inputs", "34-wide"]),
            (["--dynamic_param", bad_dyn], ValueError, ["--dynamic_param"]),
            (["--x_starts", "0"], ValueError, ["--x_starts"])):
        _refused(tmp_path, ok + flags, monkeypatch, exc, words)
    _refused(tmp_path, ["--ETG_path", CPG], monkeypatch, ValueError, ["--load"])


def test_a_table_of_steps_plus_one_rows_is_accepted(tmp_path):
    from paddlerobotics_b200 import deploy_test
    exact = str(tmp_path / "exact.npy"); np.save(exact, np.zeros((101, 12)))
    table, sd = deploy_test.check_args(deploy_test.parser().parse_args(["--load", STUDENT, "--ETG_path", exact, "--sensor_footpose", "1",
                                                                         "--RNN_mode", "GRU", "--timesteps", "0"]))
    assert table.shape == (101, 12) and sd["actor_model.l1.weight"].shape[1] == 46


def test_batch_layout():
    from paddlerobotics_b200 import deploy_test
    g, x = deploy_test.batch_layout(1, 1)
    assert g.tolist() == [0] and x.tolist() == [0.0]
    g, x = deploy_test.batch_layout(3, 5)
    assert g.tolist() == [0] * 5 + [1] * 5 + [2] * 5
    assert np.allclose(x, np.tile([-0.1, -0.05, 0.0, 0.05, 0.1], 3), rtol=0, atol=1e-15)
    assert g[0] == 0 and x[0] == -0.1           # env 0: first group, first offset


def test_group_rows(tmp_path):
    from paddlerobotics_b200 import deploy_test
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict
    rows, labels = deploy_test.group_rows([])
    assert labels == ["nominal"] and np.array_equal(rows, dynamic_dict_to_row(None)[None])
    v = np.random.default_rng(0).uniform(-1, 1, 48)
    p = str(tmp_path / "p.npy"); np.save(p, v)
    rows, labels = deploy_test.group_rows([p, "nominal"])
    assert labels == [p, "nominal"]
    assert np.array_equal(rows[0], dynamic_dict_to_row(param2dynamic_dict(v))) and np.array_equal(rows[1], dynamic_dict_to_row(None))


def test_summarise_reduces_per_group():
    from paddlerobotics_b200 import deploy_test
    group, _ = deploy_test.batch_layout(2, 3)
    res = {"fall": np.array([1, 0, 0, 1, 1, 0], bool), "length": np.array([10, 100, 100, 5, 7, 100]),
           "distance": np.arange(6.0), "velx": np.arange(6.0) / 10, "success": np.linspace(0, 1, 6)}
    a, b = deploy_test.summarise(res, group, ["nominal", "p.npy"])
    assert a == {"dynamic_param": "nominal", "envs": 3, "falls": 1, "mean_length": 70.0, "min_length": 10, "mean_distance": 1.0,
                 "mean_velx": pytest.approx(0.1), "success_rate": pytest.approx(0.2)}
    assert b["dynamic_param"] == "p.npy" and b["falls"] == 2 and b["min_length"] == 5 and b["mean_length"] == pytest.approx(112 / 3)
