"""One control step of the float32 product kernel against the float64 build from the same states, at the bench's batch size.

4096 mid-gait states (the bench workload's ETG and +-0.3 residuals, 15 control steps from the settled pose, float64) are rounded to
float32 and loaded with set_state into freshly reset float32 and float64 handles, which then take one step with the same action.  Both
builds run the same code, so their difference is the float32 rounding of one control step (13 substeps of 23 Gauss-Seidel sweeps) over
thousands of contact configurations at once, where the per-feature parity tests drive one robot.

Each bound is about 4x the largest error measured on an H100 80GB HBM3 (700 W power limit) over seeds 0-2; the measured value sits
beside it.  Relative errors are scaled by max(1, |float64|) per element; done flags are exact."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 4096
# quantity -> (bound, measured worst element over the batch)
BOUNDS = {"obs": (1.5e-3, 3.7e-4), "reward": (5e-4, 1.1e-4), "state": (1.7e-3, 4.2e-4)}


def etg():
    from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    return w, b


def mid_gait_states(seed=0, steps=15):
    """[N,37] float64 states: the settled batch after `steps` control steps of the bench's residual policy, no reset in between."""
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg()
    env = VecQuadrupedalEnv(N, precision="f64")
    env.reset(w, b)
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    for _ in range(steps):
        env.step(torch.rand(N, 12, device="cuda", dtype=torch.float64, generator=g) * 0.6 - 0.3)
    s = env.get_state().cpu().numpy()
    env.close()
    return s


def one_step(states32, action32, precision):
    """Resets a handle of the given precision, loads the float32-rounded states, takes one step; float64 numpy results."""
    import torch
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg()
    env = VecQuadrupedalEnv(N, precision=precision)
    env.reset(w, b)
    env.set_state(torch.as_tensor(states32.astype(np.float64), dtype=env.dtype, device="cuda"))
    ob, rw, dn, _ = env.step(torch.as_tensor(action32.astype(np.float64), dtype=env.dtype, device="cuda"))
    out = {"obs": ob.double().cpu().numpy(), "reward": rw.double().cpu().numpy(), "done": dn.cpu().numpy().copy(),
           "state": env.get_state().double().cpu().numpy()}
    env.close()
    return out


def rel_err(a, ref):
    return float(np.max(np.abs(a - ref) / np.maximum(1.0, np.abs(ref))))


def compare(seed=0):
    s32 = mid_gait_states(seed).astype(np.float32)
    a32 = np.random.default_rng(seed).uniform(-0.3, 0.3, (N, 12)).astype(np.float32)
    r32, r64 = one_step(s32, a32, "f32"), one_step(s32, a32, "f64")
    errs = {k: rel_err(r32[k], r64[k]) for k in ("obs", "reward", "state")}
    return errs, r32, r64


def test_f32_step_matches_f64_step_from_the_same_states():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    errs, r32, r64 = compare(0)
    assert np.isfinite(r64["obs"]).all() and np.isfinite(r64["state"]).all()
    assert np.array_equal(r32["done"], r64["done"])
    for k, (bound, _) in BOUNDS.items():
        assert errs[k] <= bound, (k, errs[k], bound)
