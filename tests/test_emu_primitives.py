"""The step kernel's scalar primitives through their HOST branches (tests/emu compiles b2q_math.cuh / b2q_sim.cuh for the CPU), against
float64 references on sampled inputs.  On the host m_rcp is 1.0f / x and m_rsqrt is 1.0f / sqrtf(x); m_sincos, Philox and the templated
kinematics, terrain and 6x6 solves are the device's source compiled for the CPU.  tests/test_gpu_primitives.py runs the device branches
exhaustively and lists where the two differ.

Bounds are about 4x the maxima measured here (x86-64, g++ -O2 -ffp-contract=off), with the measured value beside each."""
import os
import sys

import numpy as np
import pytest

import prim_ref as R

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu as E  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def _build():
    E.lib()


def sincos_samples(n=1_000_000, seed=0):
    """Uniform in [-8 pi, 8 pi], the multiples of pi/2 there and their float32 neighbours, and tiny / subnormal arguments."""
    rng = np.random.default_rng(seed)
    k = np.arange(-16, 17) * (np.pi / 2)
    near = np.concatenate([np.nextafter(np.float32(k), np.float32(np.inf)), np.float32(k), np.nextafter(np.float32(k), np.float32(-np.inf))])
    tiny = np.float32([1e-45, -1e-45, 1e-39, 1e-30, 1e-10, -1e-5])
    return np.concatenate([rng.uniform(-8 * np.pi, 8 * np.pi, n).astype(np.float32), near, tiny])


def test_host_sincos_within_its_bound():
    a = sincos_samples()
    s, c = E.sincos(a)
    es, ec = R.ulp_err(s, np.sin(a.astype(np.float64))), R.ulp_err(c, np.cos(a.astype(np.float64)))
    print("host m_sincos on %d samples in [-8pi, 8pi]: sin %.3f ulp, cos %.3f ulp" % (a.size, es.max(), ec.max()))
    assert es.max() <= 2.0 and ec.max() <= 2.0            # measured 1.47 / 1.46 ulp; the device computes the same bits (test_gpu_primitives)
    s, c = E.sincos(np.float32([np.nan, np.inf, -np.inf]))
    assert np.isnan(s).all() and np.isnan(c).all()


def test_host_rcp_and_rsqrt_are_correctly_rounded_divisions():
    rng = np.random.default_rng(1)
    bits = rng.integers(0x00800000, 0x7F800000, 1_000_000, dtype=np.uint32)
    x = bits.view(np.float32) * np.float32(rng.choice([-1, 1], bits.size))
    assert np.array_equal(E.unary(0, x), np.float32(1) / x)
    xp = np.abs(x)
    r = E.unary(1, xp)
    assert np.array_equal(r, np.float32(1) / np.sqrt(xp))
    e = R.ulp_err(r, 1 / np.sqrt(xp.astype(np.float64)))
    print("host m_rsqrt: %.3f ulp" % e.max())
    assert e.max() <= 2.0                                   # two roundings: measured 1.48 ulp


def test_host_philox_matches_the_published_definition():
    # Random123's known-answer vector for Philox4x32-10 (counter 0, key 0)
    assert E.philox4(np.zeros(1, np.uint64), np.zeros((1, 3), np.uint32)).tolist() == [[0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]]
    seeds, ctr, key = R.philox_inputs(200_000)
    ctr4 = np.concatenate([ctr, np.zeros((ctr.shape[0], 1), np.uint32)], 1)
    words = R.philox4x32_10(ctr4, key)
    assert np.array_equal(E.philox4(seeds, ctr), words)
    ref, rad = R.box_muller64(words)
    nd = E.philox_normal4(1, seeds, ctr)
    nf = E.philox_normal4(0, seeds, ctr).astype(np.float64)
    scale = np.maximum(1.0, np.repeat(rad, 2, axis=1))
    ed = float(np.max(np.abs(nd - ref) / scale) / R.EPS64)
    ef = float(np.max(np.abs(nf - ref)))
    print("host philox_normal4: double %.2f eps64 x max(1, radius), float %.3g absolute" % (ed, ef))
    assert ed <= 4                                          # measured 0.99 eps64
    assert ef <= 6e-5                                       # measured 1.4e-5 on these samples (the device sweep finds the worst case)


@pytest.mark.parametrize("prec", [0, 1])
def test_host_kinematics(prec):
    m = R.check_kinematics(E, prec, m=12, n_ik=3000)
    print("host kinematics prec %d:" % prec, m)
    assert m["nan_violations"] == 0
    if prec:
        assert m["fk"] <= 1e-13 and m["ik_interior"] <= 1e-13 and m["ik_boundary"] <= 1e-13    # measured 1.1e-16, 0, 0
    else:
        # measured 7.7e-8, 9.6e-6, and 4.4e-2 within 1e-3 of the acos / asin edge (d acos / dx is 1 / sqrt(1 - x^2))
        assert m["fk"] <= 3e-7 and m["ik_interior"] <= 3.6e-5 and m["ik_boundary"] <= 0.18


@pytest.mark.parametrize("prec", [0, 1])
def test_host_quat_to_rpy(prec):
    m = R.check_rpy(E, prec, n=8000)
    print("host quat_to_rpy prec %d:" % prec, m)
    if prec:
        assert max(m["angles"], m["rotation"], m["gimbal_rotation_scaled"], m["pitch_in_gimbal"]) <= 1e-12   # measured 0: libm, as the oracle
    else:
        # measured 3.2e-5, 3.0e-5, 4.9e3 eps32 / cos(pitch), 3.6e-4 (asin at 1: sqrt(eps32))
        assert m["angles"] <= 1.3e-4 and m["rotation"] <= 1.2e-4 and m["gimbal_rotation_scaled"] <= 2e4 and m["pitch_in_gimbal"] <= 1.5e-3


@pytest.mark.parametrize("prec", [0, 1])
def test_host_terrain(prec):
    m = R.check_terrain(E, prec)
    print("host terrain_height prec %d:" % prec, m)
    # vs_hf_height: the kernel clamps the far edges at n - 1.000001, hf_height at n - 1: 1e-6 of a cell's rise (<= 0.6 here)
    if prec:
        assert m["height"] <= 2.2e-16 and m["normal"] <= 1.3e-15 and m["vs_hf_height"] <= 1e-6        # measured 0, 3.3e-16, 5.8e-7
    else:
        assert m["height"] <= 2e-7 and m["normal"] <= 1.7e-6 and m["vs_hf_height"] <= 7e-6           # measured 4.7e-8, 4.3e-7, 1.8e-6


@pytest.mark.parametrize("prec", [0, 1])
def test_host_spd_solve(prec):
    m = R.check_solve(E, prec)
    print("host chol6/fwd6/bwd6 prec %d:" % prec, m)
    assert m["synthetic"] <= 6 and m["schur"] <= 6             # kappa up to 1e6 / 830; measured 0.38 / 0.0097 (f32), 0.34 / 1.4 (f64)
