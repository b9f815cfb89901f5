"""Camera images on the GPU (b2q_render, include/b2q_render.h) against the NumPy reference ray-caster (render_ref.py), and the
`train.py --eval 1` path that writes them."""
import json
import struct

import numpy as np
import pytest
import torch

import render_ref as RR
from paddlerobotics_b200 import render
from paddlerobotics_b200.terrain import make_terrain

pytestmark = pytest.mark.gpu
W, H = 96, 72


def _terrains():
    rng = np.random.default_rng(11)
    return {"plane": None, "stairstair": make_terrain("stairstair"), "slopeslope": make_terrain("slopeslope"),
            "balancebeam": make_terrain("balancebeam"), "rough": (rng.uniform(0, 0.03, (40, 40)), -1.0, -1.0, 0.05)}


TERRAINS = _terrains()


def make_env(n, precision, hf):
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    return VecQuadrupedalEnv(n, precision=precision, heightfield=hf)


def render_rows(env, state, ids, views, projs, w=W, h=H):
    """b2q_render on explicit state rows: returns (rc, rgba, depth, seg) as numpy."""
    V = len(ids)
    dev = env.device
    ids_t = torch.as_tensor(np.asarray(ids, dtype=np.int32), device=dev)
    v = torch.as_tensor(np.asarray(views, dtype=np.float32).reshape(V, 16), device=dev)
    p = torch.as_tensor(np.asarray(projs, dtype=np.float32).reshape(V, 16), device=dev)
    rgba = torch.zeros(V, h, w, 4, dtype=torch.uint8, device=dev)
    depth = torch.zeros(V, h, w, dtype=torch.float32, device=dev)
    seg = torch.zeros(V, h, w, dtype=torch.int32, device=dev)
    st = torch.as_tensor(state, dtype=env.dtype, device=dev).contiguous()
    rc = env.lib.b2q_render(env.h, st.data_ptr(), ids_t.data_ptr(), V, v.data_ptr(), p.data_ptr(), w, h, rgba.data_ptr(), depth.data_ptr(),
                              seg.data_ptr(), env._stream())
    torch.cuda.synchronize()
    return rc, rgba.cpu().numpy(), depth.cpu().numpy(), seg.cpu().numpy()


def cameras(pos, k):
    if k % 2 == 0:
        return render.follow_camera(pos, W, H)
    return (render.compute_view_matrix(pos + np.array([-0.6, -0.9, 0.8]), pos + np.array([0.9, 0.1, 0.0]), (0, 0, 1)),
            render.compute_projection_matrix_fov(70, W / H, 0.1, 100))


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("terrain", sorted(TERRAINS))
def test_live_handle_matches_reference(etg_shipped, precision, terrain):
    """State rows of b2q_get_state after reset and after 50 steps of the shipped gait, several envs (different env_ids) in one launch."""
    hf = TERRAINS[terrain]
    env = make_env(4, precision, hf)
    w, b = etg_shipped
    offs = np.array([0.0, 0.05, -0.05, 0.1])
    env.reset(w, b, x_offset=offs)
    for phase in ("reset", "stride"):
        if phase == "stride":
            zero = torch.zeros(4, 12, dtype=env.dtype, device=env.device)
            for _ in range(50):
                env.step(zero)
        state = env.get_state().double().cpu().numpy()
        ids = [2, 0, 3]
        cams = [cameras(state[e, :3], k) for k, e in enumerate(ids)]
        rc, rgba, depth, seg = render_rows(env, state, ids, [c[0] for c in cams], [c[1] for c in cams])
        assert rc == 0
        for k, e in enumerate(ids):
            ref = RR.render(state[e], cams[k][0], cams[k][1], W, H, hf)
            msgs = RR.compare((rgba[k], depth[k], seg[k]), ref, 0.1, 100)
            assert not msgs, (phase, e, msgs)
            assert (seg[k] >= 1).sum() > 50
    # the device API: the follow camera of every env, one launch
    rgba, depth, seg = env.get_camera_image(W, H)
    state = env.get_state().double().cpu().numpy()
    for e in range(4):
        v, p = render.follow_camera(state[e, :3], W, H)
        assert not RR.compare((rgba[e].cpu().numpy(), depth[e].cpu().numpy(), seg[e].cpu().numpy()), RR.render(state[e], v, p, W, H, hf), 0.1, 100)
    env.close()


@pytest.mark.parametrize("terrain", ["stairstair", "slopeslope", "balancebeam", "rough"])
def test_terrain_heights_top_down(terrain):
    """Orthographic top-down camera: on every terrain pixel, eye_z - linear depth equals the terrain height at the pixel centre
    within 1e-5 m, inside the grid and on its edge-clamped extension."""
    hf = TERRAINS[terrain]
    field, x0, y0, cell = hf
    env = make_env(1, "f32", hf)
    state = env.get_state().double().cpu().numpy()
    xs = (x0 - 1.0, x0 + cell * (field.shape[1] - 1) + 1.0)
    ys = (y0 - 0.7, y0 + cell * (field.shape[0] - 1) + 0.7)
    eye = np.array([0.5 * (xs[0] + xs[1]), 0.5 * (ys[0] + ys[1]), 3.0])
    view = render.compute_view_matrix(eye, eye - np.array([0, 0, 1.0]), (0, 1, 0))
    near, far = 0.1, 10.0
    hw, hh = 0.5 * (xs[1] - xs[0]), 0.5 * (ys[1] - ys[0])
    proj = [1 / hw, 0, 0, 0, 0, 1 / hh, 0, 0, 0, 0, -2 / (far - near), 0, 0, 0, -(far + near) / (far - near), 1]
    w, h = 320, 200
    rc, _, depth, seg = render_rows(env, state, [0], [view], [proj], w, h)
    assert rc == 0
    terr = seg[0] == 0
    assert terr.mean() > 0.95
    px = xs[0] + (np.arange(w) + 0.5) / w * (xs[1] - xs[0])
    py = ys[1] - (np.arange(h) + 0.5) / h * (ys[1] - ys[0])
    X, Y = np.meshgrid(px, py)
    z = eye[2] - RR.linear_depth(depth[0], near, far, ortho=True)
    err = np.abs(z - RR.hf_height(field, x0, y0, cell, X, Y))[terr]
    assert err.max() < 1e-5, err.max()
    env.close()


def test_view_independence(etg_shipped):
    """View v of a V-view launch is bit-identical to the same view rendered alone."""
    hf = TERRAINS["stairstair"]
    env = make_env(3, "f32", hf)
    env.reset(*etg_shipped)
    state = env.get_state().double().cpu().numpy()
    ids = [1, 0, 2, 1]
    cams = [cameras(state[e, :3], k) for k, e in enumerate(ids)]
    _, rgba, depth, seg = render_rows(env, state, ids, [c[0] for c in cams], [c[1] for c in cams])
    for k, e in enumerate(ids):
        _, r1, d1, s1 = render_rows(env, state, [e], [cams[k][0]], [cams[k][1]])
        np.testing.assert_array_equal(rgba[k], r1[0])
        np.testing.assert_array_equal(depth[k].view(np.uint32), d1[0].view(np.uint32))
        np.testing.assert_array_equal(seg[k], s1[0])
    env.close()


def test_graph_capture(etg_shipped):
    """A CUDA-graph capture of get_camera_image replays to identical images."""
    env = make_env(8, "f32", TERRAINS["stairstair"])
    env.reset(*etg_shipped)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = [t.clone() for t in env.get_camera_image(64, 48)]       # warm-up: buffers, constants
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        bufs = env.get_camera_image(64, 48)
    for t in bufs:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(bufs, out):
        assert torch.equal(a, b)
    assert (out[2] >= 1).any()
    env.close()


def test_bad_inputs(etg_shipped):
    hf = TERRAINS["stairstair"]
    env = make_env(2, "f32", hf)
    env.reset(*etg_shipped)
    state = env.get_state().double().cpu().numpy()
    v, p = render.follow_camera(state[0, :3], W, H)
    nan = state.copy()
    nan[0, 15] = np.nan
    far = state.copy()
    far[0, 0] += 1000.0                        # the robot out of view: the background alone
    rc, rgba, depth, seg = render_rows(env, nan, [0], [v], [p])
    assert rc == 0
    _, rgba_b, depth_b, seg_b = render_rows(env, far, [0], [v], [p])
    assert (seg <= 0).all() and (seg == 0).any()
    np.testing.assert_array_equal(rgba, rgba_b)
    np.testing.assert_array_equal(depth, depth_b)
    np.testing.assert_array_equal(seg, seg_b)
    for bad_id in (-1, 2, 1 << 30):
        rc, rgba, depth, seg = render_rows(env, state, [bad_id, 1], [v, v], [p, p])
        assert rc == 0
        assert (seg[0] == -1).all() and (depth[0] == 1).all() and (rgba[0][..., :3] == np.array(RR.SKY)).all() and (rgba[0][..., 3] == 255).all()
        assert (seg[1] >= 1).any()
    fn = env.lib.b2q_render
    st = torch.as_tensor(state, dtype=env.dtype, device=env.device)
    ids = torch.zeros(1, dtype=torch.int32, device=env.device)
    m = torch.as_tensor(np.asarray(v, np.float32), device=env.device)
    out = torch.zeros(H * W * 4, dtype=torch.uint8, device=env.device)
    ok = (st.data_ptr(), ids.data_ptr(), 1, m.data_ptr(), m.data_ptr(), W, H)
    for k, val in ((2, 0), (2, -3), (5, 0), (6, 0), (5, -1), (0, None), (1, None), (3, None), (4, None)):
        args = list(ok)
        args[k] = val
        assert fn(env.h, *args, out.data_ptr(), None, None, env._stream()) == -1, (k, val)
    assert b"b2q_render" in env.lib.b2q_last_error(env.h)
    env.close()


def _png_size(path):
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n" and data[12:16] == b"IHDR"
    w, h = struct.unpack(">II", data[16:24])
    return w, h


def test_eval_mode_writes_frames(tmp_path, capsys):
    """train.py --eval 1: a fresh checkpoint evaluated with and without --render_dir gives identical JSON metrics, and one PNG of the
    requested size per control step."""
    from paddlerobotics_b200 import train
    from paddlerobotics_b200.agent import MujocoAgent
    from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
    agent = MujocoAgent(49, 12, seed=3)
    pt = str(tmp_path / "itr_0.pt")
    agent.save(pt)
    layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
    np.savez(str(tmp_path / "itr_0.npz"), w=w, b=b, param=np.zeros(12))
    frames = tmp_path / "frames"
    base = ["--eval", "1", "--load", pt, "--task_mode", "stairstair", "--eval_envs", "2"]
    rec_frames = train.main(base + ["--render_dir", str(frames), "--render_width", "80", "--render_height", "60"])
    rec_plain = train.main(base)
    assert rec_frames == rec_plain
    lines = [json.loads(l) for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    assert lines[-1] == rec_plain
    n = len(list(frames.iterdir()))
    assert 1 <= n <= 601
    for k in (1, n):
        assert _png_size(str(frames / ("img%d.png" % k))) == (80, 60)
    assert set(rec_plain["terms"]) == {"torso", "feet", "up", "tau", "badfoot", "footcontact"}
    assert 1 <= rec_plain["mean_length"] <= 601
