"""The Bezier gait of deployment/test.py --gait 1 without a device: the per-env arithmetic the kernel runs (csrc/b2q_bezier.h, compiled
for the CPU by bezier_host.py) against the reference's own BezierGait / BezierStepper / A1 kinematics (tests/golden/bezier_gait.npz,
written by tests/golden/make_bezier_golden.py), and the deploy_bezier command: what it refuses before any device work and what it runs."""
import os

import numpy as np
import pytest

import bezier_host as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
STUDENT = os.path.join(GOLDEN, "StairStair3_BC1_itr_500383.pt")
CPG = os.path.join(GOLDEN, "gait_action_list_CPG_stairstair7_12_3.npy")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "bezier_gait.npz")))


def test_fixture_reaches_every_branch(golden):
    """The cases take each discrete path of the gait: the five held steps, touchdowns from contact and from SwRef >= 0.999, the
    reference leg in stance and in swing, and unreachable feet (NaN joint angles)."""
    td, sw, swref, ang = golden["td"], golden["swing"], golden["swref"], golden["ang"]
    assert golden["q"].shape == (27, 12) and td.shape == (27, 300)
    assert (golden["feet"][:, :5] == golden["tb0"][:, None]).all()           # timesteps <= 5: the reset feet
    assert (sw == 0).any() and (sw == 1).any() and (swref >= 0.999).any()
    assert td[0].sum() < td[1].sum()                                         # all-1 contacts set TD more often than all-0
    assert np.isnan(ang).any() and np.isfinite(ang).any()


def test_host_gait_matches_the_reference(golden):
    """Every step of every case: feet, T_b0 and joint angles within 1e-12 with NaN exactly where the reference has it; TD, the stance/swing
    flag and SwRef >= 0.999 exactly."""
    tb0, feet, ang, fl = H.rollout(golden["q"], golden["contact"])
    assert np.abs(tb0 - golden["tb0"]).max() <= 1e-12
    for got, ref in ((feet, golden["feet"]), (ang, golden["ang"])):
        assert np.array_equal(np.isnan(got), np.isnan(ref))
        ok = ~np.isnan(ref)
        err = np.abs(got[ok] - ref[ok]).max()
        print("host gait vs reference: max |diff| %.3g" % err)
        assert err <= 1e-12
    assert np.array_equal(fl[..., 0], golden["td"])
    assert np.array_equal(fl[..., 2], golden["swing"])
    assert np.array_equal(fl[..., 1] >= 0.999, golden["swref"] >= 0.999)
    assert np.abs(fl[..., 1] - golden["swref"]).max() <= 1e-12


def test_state_width_and_ik():
    from paddlerobotics_b200 import deploy
    assert H.lib().bez_state_dim() == deploy.BEZIER_STATE_DIM == 18
    pose = np.array([0, 0.9, -1.8] * 4)
    tb0, _, _, _ = H.rollout(pose[None], np.zeros((1, 1)))
    assert np.abs(H.ik(tb0[0]) - pose).max() <= 1e-12                       # IK inverts the FK that gave T_b0


def test_contact_column():
    from paddlerobotics_b200 import deploy

    def env(dis, contact):
        class _Env:
            class cfg:
                sensor_dis = dis
                sensor_contact = contact
        return _Env
    assert deploy.contact_col_of(env(0, 1)) == 0 and deploy.contact_col_of(env(1, 1)) == 3
    with pytest.raises(ValueError, match="sensor_contact"):
        deploy.contact_col_of(env(1, 0))


def _patch(monkeypatch, env, rehearse):
    from paddlerobotics_b200 import deploy_bezier, deploy_test
    for m in (deploy_bezier, deploy_test):
        monkeypatch.setattr(m, "VecQuadrupedalEnv", env)
        monkeypatch.setattr(m, "rehearse", rehearse)


def _refused(flags, monkeypatch, exc, words):
    import torch
    from paddlerobotics_b200 import deploy_bezier

    def no_device(*a, **k):
        raise AssertionError("device touched before the input check")
    monkeypatch.setattr(torch.cuda, "_lazy_init", no_device)
    _patch(monkeypatch, no_device, no_device)
    with pytest.raises(exc) as e:
        deploy_bezier.main(flags)
    for w in words:
        assert w in str(e.value), (w, str(e.value))


def test_gait_refusals_before_any_device_work(tmp_path, monkeypatch):
    """deploy_bezier refuses the gait with --sensor_contact 0 or with the action filter, and keeps deploy_test's own refusals."""
    ok = ["--load", STUDENT, "--ETG_path", CPG]
    short = str(tmp_path / "short.npy"); np.save(short, np.zeros((100, 12)))
    for flags, exc, words in (
            (["--sensor_contact", "0"], ValueError, ["--gait 1", "--sensor_contact 0", "FootContactSensor"]),
            (["--gait", "3", "--sensor_contact", "0"], ValueError, ["--gait 3"]),
            (["--enable_action_filter", "1"], NotImplementedError, ["--gait 1", "--enable_action_filter"]),
            (["--RNN_mode", "stack"], NotImplementedError, ["--RNN_mode", "--timesteps"]),
            (["--dt", "0.02"], ValueError, ["--dt"]),
            (["--ETG_path", short], ValueError, ["--ETG_path", "100 rows", "row 100"]),
            (["--sensor_dis", "1"], ValueError, ["--load", "46 inputs", "49-wide"]),
            (["--x_starts", "0"], ValueError, ["--x_starts"])):
        _refused(ok + flags, monkeypatch, exc, words)
    _refused(["--ETG_path", CPG], monkeypatch, ValueError, ["--load"])


@pytest.mark.parametrize("gait", [None, "0", "1", "2"])
def test_gait_flag_reaches_the_rehearsal(tmp_path, monkeypatch, gait):
    """deploy_bezier runs the gait by default and for any non-zero --gait (test.py's `if gait:`), and marks its records; --gait 0 is
    deploy_test, whose records are unchanged."""
    from paddlerobotics_b200 import agent, deploy_bezier
    seen = {}

    class _Env:
        def __init__(self, n, **cfg):
            seen["n"], seen["cfg"] = n, cfg

        def close(self):
            pass

    class _Student:
        def __init__(self, *a):
            pass

        def load_state_dict(self, sd):
            pass

    def fake_rehearse(env, student, table, steps, act_bound, x_offset, gait=False):
        seen["gait"] = gait
        n = seen["n"]
        return {"fall": np.zeros(n, bool), "length": np.full(n, steps), "distance": np.zeros(n), "velx": np.zeros(n), "success": np.zeros(n),
                "obs": np.zeros((steps, 46)), "action": np.zeros((steps, 12))}
    _patch(monkeypatch, _Env, fake_rehearse)
    monkeypatch.setattr(agent, "MujocoAgent", _Student)
    monkeypatch.chdir(tmp_path)
    on = gait != "0"
    recs, _ = deploy_bezier.main(["--load", STUDENT, "--ETG_path", CPG] + ([] if gait is None else ["--gait", gait]))
    assert seen["gait"] is on and seen["cfg"]["etg_enabled"] == 0 and seen["cfg"]["sensor_contact"] == 1
    assert ("gait" in recs[0]) is on and recs[0].get("gait", 1) == 1
    assert (tmp_path / "data" / "exp0_rpm.npz").exists()
