"""Camera images without a GPU: the ray-caster's device code (b2q_render.cuh) compiled for the CPU (tests/emu/emu_render.cpp) against
the independent NumPy reference (render_ref.py), the reference's own kinematics against the float64 oracle, and the small helpers of
paddlerobotics_b200/render.py (camera matrices, PNG writer)."""
import ctypes as C
import math
import os
import struct
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

import render_ref as RR
from oracle import oracle as O
from paddlerobotics_b200 import render
from paddlerobotics_b200.terrain import make_terrain

EMU_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
W, H = 96, 72
_emu = None
_emu_dir = None


def emu_lib():
    """The emulation library (tests/emu/render.mk), built into a temporary directory: the source tree may be read-only."""
    global _emu, _emu_dir
    if _emu is None:
        _emu_dir = tempfile.TemporaryDirectory(prefix="b2q_emu_render_")
        subprocess.check_call(["make", "-C", EMU_DIR, "-s", "-f", "render.mk", "OUT=" + _emu_dir.name])
        _emu = C.CDLL(os.path.join(_emu_dir.name, "libb2q_emu_render.so"))
    return _emu


def emu_render(state, view, proj, hf=None, w=W, h=H):
    lib = emu_lib()
    rgba = np.zeros((h, w, 4), np.uint8)
    depth = np.zeros((h, w), np.float32)
    seg = np.zeros((h, w), np.int32)
    st = None if state is None else np.ascontiguousarray(state, dtype=np.float64)
    v, p = np.ascontiguousarray(view, dtype=np.float32), np.ascontiguousarray(proj, dtype=np.float32)
    if hf is None:
        field, nx, ny, x0, y0, cell = None, 0, 0, 0.0, 0.0, 1.0
    else:
        field = np.ascontiguousarray(hf[0], dtype=np.float64)
        ny, nx = field.shape
        x0, y0, cell = hf[1], hf[2], hf[3]
    ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = lib.emu_render(ptr(st), C.c_double(0.02), ptr(field), nx, ny, C.c_double(x0), C.c_double(y0), C.c_double(cell), ptr(v), ptr(p), w, h,
                        ptr(rgba), ptr(depth), ptr(seg))
    assert rc == 0
    return rgba, depth, seg


@pytest.fixture(scope="module")
def oracle_states(etg_shipped):
    """settled pose, a mid-stride state of the shipped gait, and a fallen robot lying on its side (all from the float64 oracle)."""
    w, b = etg_shipped
    o = O.OracleEnv()
    o.reset(w, b)
    settled = o.get_state()
    traj = []
    for _ in range(40):
        o.step(np.zeros(12))
        traj.append(o.get_state())
    f = O.OracleEnv()
    f.reset(w, b)
    s = f.get_state()
    s[2] += 0.1
    s[3:7] = [math.sin(0.6), 0.0, 0.0, math.cos(0.6)]     # rolled by 1.2 rad: it falls over
    f.set_state(s)
    for _ in range(40):
        f.step(np.zeros(12))
    return {"settled": settled, "stride": traj[17], "fallen": f.get_state(), "traj": traj, "oracle": o}


def test_reference_kinematics_match_oracle(etg_shipped):
    w, b = etg_shipped
    o = O.OracleEnv()
    o.reset(w, b)
    for k in range(60):
        np.testing.assert_allclose(RR.toe_world(o.get_state()), o.foot_world(), rtol=0, atol=1e-12)
        o.step(np.zeros(12))


def _terrains():
    rng = np.random.default_rng(7)
    rough = (rng.uniform(0, 0.03, (40, 40)), -1.0, -1.0, 0.05)     # draw_feature_combo's random rough field
    return {"plane": None, "stairstair": make_terrain("stairstair"), "slopeslope": make_terrain("slopeslope"),
            "balancebeam": make_terrain("balancebeam"), "rough": rough}


TERRAINS = _terrains()


def _cameras(pos):
    v1, p1 = render.follow_camera(pos, W, H)
    v2 = render.compute_view_matrix(pos + np.array([-0.6, -0.9, 0.8]), pos + np.array([0.9, 0.1, 0.0]), (0, 0, 1))
    return [(v1, p1), (v2, render.compute_projection_matrix_fov(70, W / H, 0.1, 100))]


@pytest.mark.parametrize("terrain", sorted(TERRAINS))
@pytest.mark.parametrize("pose", ["settled", "stride", "fallen"])
def test_emulated_kernel_matches_reference(oracle_states, terrain, pose):
    st = oracle_states[pose]
    hf = TERRAINS[terrain]
    for view, proj in _cameras(st[:3]):
        got = emu_render(st, view, proj, hf)
        ref = RR.render(st, view, proj, W, H, hf)
        msgs = RR.compare(got, ref, 0.1, 100)
        assert not msgs, msgs
        assert (ref[2] >= 1).sum() > 50, "the robot should be in view"


def test_emulated_kernel_terrain_heights_top_down():
    """Orthographic top-down camera: on every terrain pixel, eye_z - linear depth is the terrain height at the pixel centre, inside
    and outside the grid (balancebeam's -0.3 m drop, the stairs' far end)."""
    for name in ("stairstair", "balancebeam", "rough"):
        hf = TERRAINS[name]
        field, x0, y0, cell = hf
        xs = (x0 - 1.0, x0 + cell * (field.shape[1] - 1) + 1.0)
        ys = (y0 - 0.7, y0 + cell * (field.shape[0] - 1) + 0.7)
        eye = np.array([0.5 * (xs[0] + xs[1]), 0.5 * (ys[0] + ys[1]), 3.0])
        view = render.compute_view_matrix(eye, eye - np.array([0, 0, 1.0]), (0, 1, 0))
        near, far = 0.1, 10.0
        hw, hh = 0.5 * (xs[1] - xs[0]), 0.5 * (ys[1] - ys[0])
        proj = [1 / hw, 0, 0, 0, 0, 1 / hh, 0, 0, 0, 0, -2 / (far - near), 0, 0, 0, -(far + near) / (far - near), 1]
        w, h = 120, 80
        _, depth, seg = emu_render(None, view, proj, hf, w, h)
        assert (seg == 0).all()
        px = xs[0] + (np.arange(w) + 0.5) / w * (xs[1] - xs[0])
        py = ys[1] - (np.arange(h) + 0.5) / h * (ys[1] - ys[0])
        X, Y = np.meshgrid(px, py)
        ht = RR.hf_height(field, x0, y0, cell, X, Y)
        z = eye[2] - RR.linear_depth(depth, near, far, ortho=True)
        assert np.abs(z - ht).max() < 1e-5, np.abs(z - ht).max()


def test_emulated_kernel_bad_inputs(oracle_states):
    st = oracle_states["settled"].copy()
    view, proj = _cameras(st[:3])[0]
    clean = emu_render(None, view, proj, TERRAINS["stairstair"])
    st[20] = np.nan
    got = emu_render(st, view, proj, TERRAINS["stairstair"])
    for a, b in zip(got, clean):
        np.testing.assert_array_equal(a, b)
    bad = list(view)
    bad[5] = np.inf
    rgba, depth, seg = emu_render(oracle_states["settled"], bad, proj, TERRAINS["stairstair"])
    assert (seg == -1).all() and (depth == 1).all() and (rgba[..., :3] == np.array(RR.SKY)).all()


def test_png_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    for shape in ((7, 5, 4), (3, 11, 3)):
        img = rng.integers(0, 256, shape, dtype=np.uint8)
        path = tmp_path / "img.png"
        render.write_png(str(path), img)
        data = path.read_bytes()
        assert data[:8] == b"\x89PNG\r\n\x1a\n"
        pos, chunks = 8, {}
        while pos < len(data):
            n, = struct.unpack(">I", data[pos:pos + 4])
            tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
            crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
            assert crc == zlib.crc32(tag + body) & 0xFFFFFFFF
            chunks[tag] = chunks.get(tag, b"") + body
            pos += 12 + n
        w, h, depth, ctype = struct.unpack(">IIBB", chunks[b"IHDR"][:10])
        assert (h, w, depth, ctype) == (shape[0], shape[1], 8, 6 if shape[2] == 4 else 2)
        raw = np.frombuffer(zlib.decompress(chunks[b"IDAT"]), np.uint8).reshape(h, 1 + w * shape[2])
        assert (raw[:, 0] == 0).all()
        np.testing.assert_array_equal(raw[:, 1:].reshape(shape), img)


def test_camera_matrices_closed_form():
    for eye, target, up in (((1.0, -2.0, 0.5), (0.2, 0.3, 0.1), (0, 0, 1)), ((0, 0, 3), (0, 0, 0), (0, 1, 0)), ((-1, 4, 2), (3, 1, -1), (0.2, 0.1, 1))):
        e, t, u = map(np.asarray, (eye, target, up))
        f = (t - e) / np.linalg.norm(t - e)
        s = np.cross(f, u) / np.linalg.norm(np.cross(f, u))
        uu = np.cross(s, f)
        M = np.eye(4)
        M[0, :3], M[1, :3], M[2, :3] = s, uu, -f
        M[:3, 3] = -M[:3, :3] @ e
        np.testing.assert_allclose(np.array(render.compute_view_matrix(eye, target, up)).reshape(4, 4).T, M, atol=1e-12)
    for fov, aspect, n, fa in ((60, 4 / 3, 0.1, 100), (45, 1.0, 0.01, 5), (90, 2.0, 1.0, 1000)):
        fcot = 1 / math.tan(math.radians(fov) / 2)
        P = np.array([[fcot / aspect, 0, 0, 0], [0, fcot, 0, 0], [0, 0, (fa + n) / (n - fa), 2 * fa * n / (n - fa)], [0, 0, -1, 0]])
        np.testing.assert_allclose(np.array(render.compute_projection_matrix_fov(fov, aspect, n, fa)).reshape(4, 4).T, P, atol=1e-12)
    # a point on the near / far plane maps to depth 0 / 1
    P = np.array(render.compute_projection_matrix_fov(60, 1.0, 0.1, 100)).reshape(4, 4).T
    for z, d in ((-0.1, 0.0), (-100.0, 1.0)):
        c = P @ np.array([0, 0, z, 1.0])
        assert abs(0.5 * c[2] / c[3] + 0.5 - d) < 1e-12
