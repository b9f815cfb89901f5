"""The step kernel's float32 device primitives and the ETG reach clip, against float64 references.

m_sincos, m_rcp and m_rsqrt run only in the float32 device build (b2q_math.cuh): the float64 build calls libm and the CPU emulation
compiles their host branches.  tests/gpu_probe runs them exhaustively over float inputs, each thread comparing with a float64 reference on
the device; it also runs both Philox implementations against the CUDA toolkit's curand_Philox4x32_10, and the kinematics, quat_to_rpy,
terrain_height and the 6x6 Cholesky solves in both precisions on the shared checks of tests/prim_ref.py.  The ETG reach clip runs through
the product handle.

Each bound is about 4x the largest value measured on an H100 80GB HBM3 (700 W power limit), with the measured value beside it; -s prints
the measured maxima."""
import os
import sys

import numpy as np
import pytest

import prim_ref as R

pytestmark = pytest.mark.gpu

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(_HERE, "gpu_probe"))
sys.path.insert(0, os.path.join(_HERE, "emu"))
import probe as P  # noqa: E402
import emu as E  # noqa: E402

TWO_PI8 = P.f32_bits(8 * np.pi)


@pytest.fixture(scope="module", autouse=True)
def _build():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    P.lib(); E.lib()


# ---- m_sincos -------------------------------------------------------------------------------------------------------------------------
# Callers: leg_kin's q1, q2 and q1 + q2 (joint angles: the URDF ranges reach |q| < 4.2 and |q1 + q2| < 6.9, a diverging state more) and
# the Euler step's half rotation angle |w| dt / 2 (< 1 for |w| < 1000 rad/s at dt = 2 ms).  [-8 pi, 8 pi] covers them with room.
def test_sincos_exhaustive_in_the_callers_range():
    es, xs, ec, xc, bad_norm = P.sweep(0, 0, TWO_PI8, True)
    print("\nm_sincos over all %d floats in [-8pi, 8pi]: sin %.3f ulp (at %r), cos %.3f ulp (at %r), s^2+c^2 off 1 by > 4 ulp: %d"
          % (2 * (TWO_PI8 + 1), es, xs, ec, xc, bad_norm))
    assert es <= 2.0 and ec <= 2.0          # measured 1.497 / 1.481 ulp
    assert bad_norm == 0


def test_sincos_reference_outside_range_and_specials():
    rng = np.random.default_rng(0)
    a = rng.uniform(-8 * np.pi, 8 * np.pi, 1_000_000).astype(np.float32)
    s, c, ds, dc = P.sincos(a)
    a64 = a.astype(np.float64)
    # the device's double sin / cos, the sweep's reference, against NumPy's
    assert np.max(np.abs(ds - np.sin(a64))) <= 4 * R.EPS64 and np.max(np.abs(dc - np.cos(a64))) <= 4 * R.EPS64
    # beyond the callers' range: |a| up to 2^20; the reduction's error grows with |a|, the outputs stay finite and on the unit circle
    big = (rng.choice([-1, 1], 200_000) * 2.0 ** rng.uniform(np.log2(8 * np.pi), 20, 200_000)).astype(np.float32)
    s, c, ds, dc = P.sincos(big)
    assert np.isfinite(s).all() and np.isfinite(c).all()
    norm = np.abs(s.astype(np.float64) ** 2 + c.astype(np.float64) ** 2 - 1) / R.EPS32
    err = max(R.ulp_err(s, ds).max(), R.ulp_err(c, dc).max())
    print("\nm_sincos for 8pi < |a| <= 2^20: worst %.3g ulp, |s^2 + c^2 - 1| <= %.2f eps32" % (err, norm.max()))
    assert norm.max() <= 4
    s, c, _, _ = P.sincos(np.float32([np.nan, np.inf, -np.inf]))
    assert np.isnan(s).all() and np.isnan(c).all()


# ---- m_rcp ----------------------------------------------------------------------------------------------------------------------------
# Callers: 1 / det of the 3x3 joint-space block (its links' masses and inertias keep det > 1e-9 and finite), 1 / W_ii of the active
# contact rows (W_ii >= the inverse effective mass of a toe, far from 0 and from 2^126), and sh / th only for th >= 1e-4.  None reaches
# 0, infinity, a subnormal or |x| > 2^126, where the device result is NaN, NaN, NaN and a signed zero.
def test_rcp_exhaustive_over_all_finite_floats():
    e, x, edge_err, xe, not_cr = P.sweep(1, 1, 0x7F7FFFFF, True)
    print("\nm_rcp over all finite nonzero floats: %.4f ulp where x and 1/x are normal (at %r); %d results differ from the correctly rounded "
          "1/x the host computes; edge values as documented: %s" % (e, x, not_cr, edge_err == 0))
    assert e <= 0.5                         # measured 0.5000: correctly rounded, as the host's 1.0f / x (and 0 of 4.2e9 results differ from it)
    assert not_cr == 0
    assert edge_err == 0, xe
    edges = np.float32([0.0, -0.0, np.inf, -np.inf, 1e-40, -1e-40, 2.0 ** 127, -(2.0 ** 127)])
    got = P.unary(0, edges)
    print("m_rcp at 0, -0, inf, -inf, 1e-40, -1e-40, 2^127, -2^127:", got.tolist())
    assert np.isnan(got[:6]).all() and got[6] == 0 and not np.signbit(got[6]) and got[7] == 0 and np.signbit(got[7])


# ---- m_rsqrt --------------------------------------------------------------------------------------------------------------------------
def test_rsqrt_exhaustive_over_positive_normal_floats():
    e, x, _, _, diff_host = P.sweep(2, 0x00800000, 0x7F7FFFFF, False)
    print("\nm_rsqrt over all positive normal floats: %.4f ulp (at %r); %d differ from the host's 1.0f / sqrtf(x)" % (e, x, diff_host))
    assert e <= 2.0                         # measured 1.5145 ulp; CUDA documents rsqrtf to 2 ulp


# ---- host vs device branches ----------------------------------------------------------------------------------------------------------
def test_host_and_device_branches_differ_only_within_the_bounds():
    rng = np.random.default_rng(3)
    a = rng.uniform(-8 * np.pi, 8 * np.pi, 2_000_000).astype(np.float32)
    sd, cd, ds, dc = P.sincos(a)
    sh, ch = E.sincos(a)
    n_sc = int(np.sum((sd.view(np.uint32) != sh.view(np.uint32)) | (cd.view(np.uint32) != ch.view(np.uint32))))
    bits = rng.integers(0x00800000, 0x7F800000, 2_000_000, dtype=np.uint32)
    x = bits.view(np.float32)
    out = {}
    for which, name, ref in ((0, "rcp", 1 / x.astype(np.float64)), (1, "rsqrt", 1 / np.sqrt(x.astype(np.float64)))):
        d, h = P.unary(which, x), E.unary(which, x)
        dif = d != h
        out[name] = dif
        print("host vs device m_%s: %d of %d samples differ; device %.3f / host %.3f ulp there"
              % (name, dif.sum(), x.size, R.ulp_err(d[dif], ref[dif]).max(initial=0), R.ulp_err(h[dif], ref[dif]).max(initial=0)))
        if which == 1:
            assert R.ulp_err(d[dif], ref[dif]).max(initial=0) <= 2.0 and R.ulp_err(h[dif], ref[dif]).max(initial=0) <= 2.0   # measured 1.51 / 1.47
    print("host vs device m_sincos: %d of %d samples differ" % (n_sc, a.size))
    assert n_sc == 0                        # the same source and the same fmaf / rintf: bit-identical
    # m_rcp: the device is correctly rounded wherever 1/x is normal, so the branches differ exactly where |x| > 2^126 (device: signed
    # zero, host: the subnormal 1/x)
    assert np.array_equal(out["rcp"], x > 2.0 ** 126)


# ---- Philox -----------------------------------------------------------------------------------------------------------------------------
def test_philox_against_curand():
    m = P.philox(100_000_000)
    print("\nPhilox over 1e8 (key, counter) tuples:", m)
    assert m["word_mismatch"] == 0 and m["normal_mismatch"] == 0, m
    # relative errors in eps x max(1, radius), against float64 from the same (float32-rounded) u: measured 0.50, 3.67, 3.44
    assert m["n4d_rel"] <= 2 and m["n4f_rel"] <= 15 and m["pn_rel"] <= 14
    # u = (r >> 8) + 0.5 rounds in float32 for r >> 8 >= 2^23; at u -> 1 the radius sqrt(-2 ln u) loses 2.4e-4 absolute at most
    assert m["n4f_abs_exact_u"] <= 5e-4 and m["pn_abs_exact_u"] <= 5e-4          # measured 2.44e-4, 2.37e-4


# ---- kinematics, quat_to_rpy, terrain, 6x6 solves ------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [0, 1])
def test_kinematics(prec):
    m = R.check_kinematics(P, prec)
    print("\ndevice kinematics prec %d:" % prec, m)
    assert m["nan_violations"] == 0
    if prec:
        # measured 1.4e-16, 3.2e-14; within 1e-3 of the acos / asin edge 1.1e-10: the device's acos and the oracle's libm differ by an ulp,
        # which 1 / sqrt(1 - x^2) amplifies
        assert m["fk"] <= 1e-13 and m["ik_interior"] <= 1e-13 and m["ik_boundary"] <= 5e-10
    else:
        assert m["fk"] <= 3e-7 and m["ik_interior"] <= 3.6e-5 and m["ik_boundary"] <= 0.18     # measured 6.2e-8, 9.1e-6, 2.2e-2


@pytest.mark.parametrize("prec", [0, 1])
def test_quat_to_rpy(prec):
    m = R.check_rpy(P, prec)
    print("\ndevice quat_to_rpy prec %d:" % prec, m)
    if prec:   # measured 2.0e-14, 1.7e-14, 1.54 eps64 / cos(pitch), 1.5e-8 (asin at 1: sqrt(eps64))
        assert m["angles"] <= 1e-13 and m["rotation"] <= 1e-13 and m["gimbal_rotation_scaled"] <= 8 and m["pitch_in_gimbal"] <= 6e-8
    else:      # measured 4.6e-5, 7.2e-5, 5.5e3 eps32 / cos(pitch), 3.4e-4
        assert m["angles"] <= 1.8e-4 and m["rotation"] <= 2.9e-4 and m["gimbal_rotation_scaled"] <= 2.2e4 and m["pitch_in_gimbal"] <= 1.5e-3


@pytest.mark.parametrize("prec", [0, 1])
def test_terrain(prec):
    m = R.check_terrain(P, prec)
    print("\ndevice terrain_height prec %d:" % prec, m)
    if prec:   # measured 5.6e-17, 3.3e-16, 5.8e-7 (the n - 1.000001 clamp: 1e-6 of a cell's rise, <= 0.6 here)
        assert m["height"] <= 2.2e-16 and m["normal"] <= 1.3e-15 and m["vs_hf_height"] <= 1e-6
    else:      # measured 4.7e-8, 4.0e-7, 1.8e-6
        assert m["height"] <= 2e-7 and m["normal"] <= 1.7e-6 and m["vs_hf_height"] <= 7e-6


@pytest.mark.parametrize("prec", [0, 1])
def test_spd_solve(prec):
    m = R.check_solve(P, prec)
    print("\ndevice chol6/fwd6/bwd6 prec %d:" % prec, m)
    assert m["synthetic"] <= 6 and m["schur"] <= 6         # kappa up to 1e6 / 830; measured 0.42 / 0.0057 (f32), 0.35 / 1.41 (f64)


# ---- the ETG reach clip through the product handle ------------------------------------------------------------------------------------
STEPS = 12


def _gaits(w, b, n_es=240, sigma=0.05, seed=0):
    """The shipped gait with W, b scaled by 1.0 .. 3.0, then Gaussian perturbations of its 63 weights at sigma, about the size of its
    largest weight (an ES-like population whose footholds often leave the leg's reach)."""
    sc = np.linspace(1.0, 3.0, 16)
    W = [w * s for s in sc]; B = [b * s for s in sc]
    rng = np.random.default_rng(seed)
    for _ in range(n_es):
        W.append(w + sigma * rng.normal(size=w.shape)); B.append(b + sigma * rng.normal(size=b.shape))
    return np.array(W), np.array(B)


def _shrink_margins(cfg, w, b, t):
    """Per leg, the float64 shrink loop of act_clip (etg.py) and the smallest |ik margin| over its tries, in eps32."""
    from oracle import oracle as O
    from paddlerobotics_b200 import etg as G
    tries, closest = np.zeros(4, int), np.zeros(4)
    for k in range(4):
        r = O.etg_features(cfg, t if k in (0, 3) else t + 0.25)
        d = w.reshape(3, 20) @ r + b
        m_min = np.inf
        for i in range(200):
            f = G.BASE_FOOT[k] + d - G.HIP_OFFSETS[k]
            m = float(R.ik_margins(f[None], np.array([k]))[0])
            m_min = min(m_min, abs(m))
            if m >= 0:
                break
            d = d * 0.95
        tries[k], closest[k] = i, m_min / R.EPS32
    return tries, closest


def test_etg_reach_clip_matches_the_oracle(etg_shipped):
    import torch
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    cfg = O.default_config()
    W, B = _gaits(*etg_shipped)
    n = W.shape[0]
    ref = np.array([[O.etg_act(cfg, W[i], B[i], k * 0.026)[0] for k in range(1, STEPS + 1)] for i in range(n)])   # [n][steps][12]
    got = {}
    for prec in ("f64", "f32"):
        env = VecQuadrupedalEnv(n, precision=prec)
        env.reset(W, B)
        rows = []
        for _ in range(STEPS):
            _, _, _, info = env.step(torch.zeros(n, 12, dtype=env.dtype, device="cuda"))
            rows.append(info[:, 12:24].double().cpu().numpy().copy())
        got[prec] = np.stack(rows, 1)
        env.close()
    clipped = np.array([[_shrink_margins(cfg, W[i], B[i], 0.026)[0].max() > 0] for i in range(n)]).ravel()
    e64 = np.abs(got["f64"] - ref)
    assert np.isfinite(ref).all()
    assert e64.max() <= 1e-12, e64.max()
    e32 = np.abs(got["f32"] - ref).max(2)               # [n][steps]
    bound = 3e-4                                        # measured 7.7e-5; a shrink step moves the target by 5 % of the foot delta
    jumps = np.argwhere(e32 > bound)
    explained = 0
    for i, k in jumps:
        tries, closest = _shrink_margins(cfg, W[i], B[i], (k + 1) * 0.026)
        assert closest.min() <= 128, (i, k, e32[i, k], tries, closest)   # a try whose float64 margin is within float32 rounding of the edge
        explained += 1
    print("\nETG reach clip: %d of %d gaits clip at t = 0.026; float64 %.2e; float32 %.2e outside %d (gait, step) pairs of %d whose shrink "
          "count differs from float64's (each with a try within 128 eps32 of the acos / asin edge)"
          % (clipped.sum(), n, e64.max(), np.where(e32 > bound, 0, e32).max(), explained, e32.size))


def test_etg_reach_clip_all_tries_nan(etg_shipped):
    """Weights no shrink can bring into reach (infinite, or 1e30): the target is NaN, the episode ends on its first step with the nan flag,
    in both precisions and in the oracle."""
    import torch
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_shipped
    W = np.array([w, w]); B = np.array([b, b])
    W[0, 0, 3] = np.inf
    W[1] *= 1e30
    for i in range(2):
        act, _ = O.etg_act(O.default_config(), W[i], B[i], 0.026)
        assert np.isnan(act).any()
        o = O.OracleEnv(O.default_config())
        o.reset(W[i], B[i])
        _, _, done, info = o.step(np.zeros(12))
        assert done and info[9] != 0
    for prec in ("f64", "f32"):
        env = VecQuadrupedalEnv(2, precision=prec)
        env.reset(W, B)
        _, _, done, info = env.step(torch.zeros(2, 12, dtype=env.dtype, device="cuda"))
        info = info.double().cpu().numpy()
        assert done.cpu().numpy().all() and (info[:, 9] != 0).all() and np.isnan(info[:, 12:24]).any(1).all(), (prec, info[:, 9])
        env.close()
