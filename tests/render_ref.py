"""Independent float64 NumPy reference of the camera-image kernel (paddlerobotics_b200/csrc/b2q_render.cuh) — test infrastructure.

* Link frames come from this module's own forward kinematics, written from the a1.py conventions (hip offsets, hip-roll about x,
  thigh and calf pitch about y, link lengths 0.2 m), not from leg_kin().  test_render_cpu.py checks the toe centres against the
  float64 oracle.
* The height field is intersected by a different algorithm from the kernel's cell-by-cell quadratic: a dense march along the ray
  (at most a quarter cell per sample) plus bisection on z_ray(t) - h(x(t), y(t)), with h restated from terrain_height() including
  its edge clamp.
* The spec constants (geometry table, colours, light) are restated from the issue's tables.

render() returns (rgba [H,W,4] uint8, depth [H,W], seg [H,W] int32, fragile [H,W] bool): `fragile` marks pixels whose result
depends on which side of a discontinuity the hit lands within 1e-4 m (a checker line, a grid line of the height field, a box or
cylinder edge), or whose ray meets the terrain almost tangentially, where float32 and float64 may legitimately differ.
"""
import numpy as np

HIP_XY = np.array([[0.183, -0.047], [0.183, 0.047], [-0.183, -0.047], [-0.183, 0.047]])
COM_OFF = np.array([-0.012731, -0.002186, -0.000515])
L_HIP, L_UP, L_LOW = 0.08505, 0.2, 0.2
TRUNK, THIGH, CALF = np.array([0.267, 0.194, 0.114]), np.array([0.034, 0.0245, 0.2]), np.array([0.016, 0.016, 0.2])
HIP_R, HIP_LEN = 0.046, 0.04
LIGHT = np.array([0.4, -0.3, 0.866025])
AMBIENT, DIFFUSE, CHECKER = 0.3, 0.7, 0.25
SKY = (178, 204, 230)
COLOURS = {0: (0.85, 0.55, 0.15), 1: (0.35, 0.35, 0.38), 2: (0.20, 0.40, 0.80), 3: (0.15, 0.15, 0.18), 4: (0.90, 0.20, 0.20),
           5: (0.70, 0.68, 0.62), 6: (0.50, 0.48, 0.44)}
EDGE = 1e-4


def rx(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def ry(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def quat_matrix(q):
    x, y, z, w = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def leg_frames(q3, leg):
    """Base-frame link frames of one leg (a1.py: hip at HIP_XY + COM offset, hip roll about x, the thigh joint l_hip out along the
    rolled y axis (negative on the right legs 0, 2), pitch about y at the thigh and knee).  Returns (p1, R1, p2, R2, p3, R3, toe)."""
    side = 1.0 if leg % 2 else -1.0
    p1 = np.array([HIP_XY[leg, 0], HIP_XY[leg, 1], 0.0]) + COM_OFF
    R1 = rx(q3[0])
    p2 = p1 + R1 @ np.array([0.0, side * L_HIP, 0.0])
    R2 = R1 @ ry(q3[1])
    p3 = p2 + R2 @ np.array([0.0, 0.0, -L_UP])
    R3 = R2 @ ry(q3[2])
    toe = p3 + R3 @ np.array([0.0, 0.0, -L_LOW])
    return p1, R1, p2, R2, p3, R3, toe


def toe_world(state):
    s = np.asarray(state, dtype=np.float64)
    R = quat_matrix(s[3:7])
    return np.array([s[:3] + R @ leg_frames(s[13 + 3 * k:16 + 3 * k], k)[6] for k in range(4)])


def primitives(state, foot_radius=0.02):
    """[(kind, centre, axes (columns), half extents, seg)] in world coordinates; kind 'box' | 'cyl' (about local y) | 'sphere'."""
    s = np.asarray(state, dtype=np.float64)
    pos, R = s[:3], quat_matrix(s[3:7])
    out = [("box", pos + R @ COM_OFF, R, TRUNK / 2, 1)]
    for k in range(4):
        p1, R1, p2, R2, p3, R3, toe = leg_frames(s[13 + 3 * k:16 + 3 * k], k)
        out.append(("cyl", pos + R @ p1, R @ R1, np.array([HIP_R, HIP_LEN / 2, HIP_R]), 2 + 4 * k))
        out.append(("box", pos + R @ (p2 + R2 @ np.array([0, 0, -0.1])), R @ R2, THIGH / 2, 3 + 4 * k))
        out.append(("box", pos + R @ (p3 + R3 @ np.array([0, 0, -0.1])), R @ R3, CALF / 2, 4 + 4 * k))
        out.append(("sphere", pos + R @ toe, R @ R3, np.full(3, foot_radius), 5 + 4 * k))
    return out


def hf_height(hf, x0, y0, cell, x, y):
    """terrain_height() restated (vectorised): bilinear inside the grid, edge-clamped outside."""
    ny, nx = hf.shape
    fx = np.clip((x - x0) / cell, 0.0, nx - 1.0)
    fy = np.clip((y - y0) / cell, 0.0, ny - 1.0)
    ix = np.minimum(np.floor(fx).astype(np.int64), nx - 2)
    iy = np.minimum(np.floor(fy).astype(np.int64), ny - 2)
    tx, ty = fx - ix, fy - iy
    return ((1 - tx) * (1 - ty) * hf[iy, ix] + tx * (1 - ty) * hf[iy, ix + 1] + (1 - tx) * ty * hf[iy + 1, ix] + tx * ty * hf[iy + 1, ix + 1])


def hf_normal(hf, x0, y0, cell, x, y):
    """Surface normal of the bilinear field and its clamped extension (zero slope along a clamped direction)."""
    ny, nx = hf.shape
    gx, gy = (x - x0) / cell, (y - y0) / cell
    fx, fy = np.clip(gx, 0.0, nx - 1.0), np.clip(gy, 0.0, ny - 1.0)
    ix = np.minimum(np.floor(fx).astype(np.int64), nx - 2)
    iy = np.minimum(np.floor(fy).astype(np.int64), ny - 2)
    tx, ty = fx - ix, fy - iy
    h00, h10, h01, h11 = hf[iy, ix], hf[iy, ix + 1], hf[iy + 1, ix], hf[iy + 1, ix + 1]
    hx = ((1 - ty) * (h10 - h00) + ty * (h11 - h01)) / cell
    hy = ((1 - tx) * (h01 - h00) + tx * (h11 - h10)) / cell
    hx = np.where((gx < 0) | (gx > nx - 1), 0.0, hx)
    hy = np.where((gy < 0) | (gy > ny - 1), 0.0, hy)
    n = np.stack([-hx, -hy, np.ones_like(hx)], -1)
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


def rays(view, proj, W, H):
    pv = np.asarray(proj, dtype=np.float64).reshape(4, 4).T @ np.asarray(view, dtype=np.float64).reshape(4, 4).T
    inv = np.linalg.inv(pv)
    xs = (2 * np.arange(W) + 1) / W - 1
    ys = 1 - (2 * np.arange(H) + 1) / H
    X, Y = np.meshgrid(xs, ys)
    def unproject(z):
        p = np.stack([X, Y, np.full_like(X, z), np.ones_like(X)], -1) @ inv.T
        return p[..., :3] / p[..., 3:]
    o, f = unproject(-1.0), unproject(1.0)
    d = f - o
    tfar = np.linalg.norm(d, axis=-1)
    return o, d / tfar[..., None], tfar, pv


def _hit_box(o, d, h):
    with np.errstate(divide="ignore", invalid="ignore"):
        t0, t1 = (-h - o) / d, (h - o) / d
    tlo, thi = np.minimum(t0, t1), np.maximum(t0, t1)
    par = d == 0
    tlo = np.where(par, np.where(np.abs(o) <= h, -np.inf, np.inf), tlo)
    thi = np.where(par, np.where(np.abs(o) <= h, np.inf, -np.inf), thi)
    tn, tf = tlo.max(-1), thi.min(-1)
    ax = tlo.argmax(-1)
    hit = (tn <= tf) & (tn > 0)
    t = np.where(hit, tn, np.inf)
    n = np.zeros_like(o)
    sgn = -np.sign(np.take_along_axis(d, ax[..., None], -1))[..., 0]
    np.put_along_axis(n, ax[..., None], sgn[..., None], -1)
    srt = np.sort(tlo, -1)
    edge = hit & ((srt[..., 2] - srt[..., 1]) < EDGE)
    return t, n, edge


def _hit_cyl(o, d, h):
    r, hl = h[0], h[1]
    a = d[..., 0] ** 2 + d[..., 2] ** 2
    b = o[..., 0] * d[..., 0] + o[..., 2] * d[..., 2]
    c = o[..., 0] ** 2 + o[..., 2] ** 2 - r * r
    with np.errstate(divide="ignore", invalid="ignore"):
        disc = b * b - a * c
        ts = (-b - np.sqrt(np.maximum(disc, 0))) / a
    ys = o[..., 1] + d[..., 1] * ts
    side = (a > 0) & (disc >= 0) & (ts > 0) & (np.abs(ys) <= hl)
    s = np.where(d[..., 1] > 0, -1.0, 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        tc = (s * hl - o[..., 1]) / d[..., 1]
    xc, zc = o[..., 0] + d[..., 0] * tc, o[..., 2] + d[..., 2] * tc
    cap = (d[..., 1] != 0) & (tc > 0) & (xc ** 2 + zc ** 2 <= r * r)
    t = np.where(side, ts, np.inf)
    usecap = cap & (tc < t)
    t = np.where(usecap, tc, t)
    p = o + d * np.where(np.isfinite(t), t, 0)[..., None]
    n = np.where(usecap[..., None], np.stack([np.zeros_like(s), s, np.zeros_like(s)], -1),
                 np.stack([p[..., 0] / r, np.zeros_like(s), p[..., 2] / r], -1))
    edge = np.isfinite(t) & ((np.abs(np.abs(p[..., 1]) - hl) < EDGE) | (np.abs(np.hypot(p[..., 0], p[..., 2]) - r) < EDGE) & usecap)
    return t, n, edge


def _hit_sphere(o, d, h):
    b = (o * d).sum(-1)
    c = (o * o).sum(-1) - h[0] ** 2
    disc = b * b - c
    t = -b - np.sqrt(np.maximum(disc, 0))
    t = np.where((disc >= 0) & (t > 0), t, np.inf)
    p = o + d * np.where(np.isfinite(t), t, 0)[..., None]
    return t, p / h[0], np.zeros(t.shape, bool)


def _march_hf(hf, x0, y0, cell, o, d, tmax):
    """First t in [0, tmax] with z(t) <= h(x(t), y(t)): dense samples a quarter cell apart, then bisection."""
    lo_h, hi_h = hf.min() - 1e-3, hf.max() + 1e-3
    with np.errstate(divide="ignore", invalid="ignore"):
        ta, tb = (hi_h - o[:, 2]) / d[:, 2], (lo_h - o[:, 2]) / d[:, 2]
    t0 = np.where(d[:, 2] == 0, np.where((o[:, 2] >= lo_h) & (o[:, 2] <= hi_h), 0.0, np.inf), np.maximum(0.0, np.minimum(ta, tb)))
    t1 = np.where(d[:, 2] == 0, tmax, np.minimum(tmax, np.maximum(ta, tb)))
    out = np.full(o.shape[0], np.inf)
    f = lambda idx, t: o[idx, 2] + d[idx, 2] * t - hf_height(hf, x0, y0, cell, o[idx, 0] + d[idx, 0] * t, o[idx, 1] + d[idx, 1] * t)
    step = 0.25 * cell
    act = np.nonzero(t0 <= t1)[0]
    f0 = f(act, t0[act])
    out[act[f0 <= 0]] = t0[act[f0 <= 0]]
    keep = f0 > 0
    act, tprev, fprev = act[keep], t0[act[keep]], f0[keep]
    fprev2 = np.full(act.shape, np.inf)

    def bisect(idx, a, b):
        for _ in range(60):
            m = 0.5 * (a + b)
            below = f(idx, m) <= 0
            b, a = np.where(below, m, b), np.where(below, a, m)
        return b

    while act.size:
        tcur = np.minimum(tprev + step, t1[act])
        fc = f(act, tcur)
        hit = fc <= 0
        # a ray that only grazes the surface between two samples: at a sampled local minimum of f, minimise f over the two steps
        # around it (ternary search) and bisect up to the minimiser when it lies below the surface
        graze = ~hit & (fprev < fprev2) & (fprev <= fc) & (fprev < step)
        if graze.any():
            gi = np.nonzero(graze)[0]
            a, b = tprev[gi] - step, tcur[gi]
            for _ in range(80):
                m1, m2 = a + (b - a) / 3, b - (b - a) / 3
                lower = f(act[gi], m1) < f(act[gi], m2)
                b, a = np.where(lower, m2, b), np.where(lower, a, m1)
            tm = 0.5 * (a + b)
            under = f(act[gi], tm) <= 0
            if under.any():
                g = gi[under]
                out[act[g]] = bisect(act[g], tprev[g] - step, tm[under])
                hit[g] = True
        if hit.any():
            h = np.nonzero(hit & ~np.isfinite(out[act]))[0]
            out[act[h]] = bisect(act[h], tprev[h], tcur[h])
        done = hit | (tcur >= t1[act])
        act, fprev2, fprev, tprev = act[~done], fprev[~done], fc[~done], tcur[~done]
    return out


def render(state, view, proj, W, H, hf=None, foot_radius=0.02):
    """state [37] or None (no robot); hf = (field [ny,nx], x0, y0, cell) or None (plane)."""
    o, d, tfar, pv = rays(view, proj, W, H)
    o, d, tfar = o.reshape(-1, 3), d.reshape(-1, 3), tfar.reshape(-1)
    n_px = o.shape[0]
    t = np.full(n_px, np.inf)
    nrm = np.zeros((n_px, 3))
    seg = np.full(n_px, -1, np.int32)
    fragile = np.zeros(n_px, bool)
    if state is not None and np.all(np.isfinite(state)):
        for kind, c, A, h, sid in primitives(state, foot_radius):
            lo, ld = (o - c) @ A, d @ A
            ti, nl, edge = {"box": _hit_box, "cyl": _hit_cyl, "sphere": _hit_sphere}[kind](lo, ld, h)
            better = (ti < t) & (ti <= tfar)
            t = np.where(better, ti, t)
            nrm = np.where(better[:, None], nl @ A.T, nrm)
            seg = np.where(better, sid, seg)
            fragile = np.where(better, edge, fragile)
    tmax = np.minimum(t, tfar)
    if hf is None:
        with np.errstate(divide="ignore", invalid="ignore"):
            tt = -o[:, 2] / d[:, 2]
        tt = np.where((d[:, 2] != 0) & (tt >= 0) & (tt <= tmax), tt, np.inf)
    else:
        tt = _march_hf(hf[0], hf[1], hf[2], hf[3], o, d, tmax)
    ter = tt < t
    t = np.where(ter, tt, t)
    seg = np.where(ter, 0, seg)
    p = o + d * np.where(np.isfinite(t), t, 0)[:, None]
    if hf is not None:
        nrm = np.where(ter[:, None], hf_normal(hf[0], hf[1], hf[2], hf[3], p[:, 0], p[:, 1]), nrm)
        gx, gy = (p[:, 0] - hf[1]) / hf[3], (p[:, 1] - hf[2]) / hf[3]
        near_grid = (np.abs(gx - np.round(gx)) * hf[3] < EDGE) | (np.abs(gy - np.round(gy)) * hf[3] < EDGE)
    else:
        nrm = np.where(ter[:, None], np.array([0.0, 0.0, 1.0]), nrm)
        near_grid = np.zeros(n_px, bool)
    cx, cy = p[:, 0] / CHECKER, p[:, 1] / CHECKER
    near_check = (np.abs(cx - np.round(cx)) * CHECKER < EDGE) | (np.abs(cy - np.round(cy)) * CHECKER < EDGE)
    # a ray that meets the terrain almost tangentially (over the crest of a bump) may or may not touch it at float32 precision
    grazing = np.abs((nrm * d).sum(-1)) < 0.05
    fragile = np.where(ter, near_grid | near_check | grazing, fragile)
    par = (np.floor(cx) + np.floor(cy)).astype(np.int64) & 1
    cls = np.where(seg == 0, 5 + par, np.where(seg == 1, 0, 1 + (seg - 2) % 4))
    leg = np.where(seg >= 2, (seg - 2) // 4, 1)
    dim = np.where((seg >= 2) & ((leg == 0) | (leg == 2)), 0.8, 1.0)
    base = np.array([COLOURS[int(c)] for c in range(7)])[np.clip(cls, 0, 6)] * dim[:, None]
    sh = AMBIENT + DIFFUSE * np.maximum(nrm @ LIGHT, 0.0)
    rgb = np.floor(np.clip(base * sh[:, None], 0, 1) * 255 + 0.5).astype(np.uint8)
    hit = seg >= 0
    rgba = np.empty((n_px, 4), np.uint8)
    rgba[:, :3] = np.where(hit[:, None], rgb, np.array(SKY, np.uint8))
    rgba[:, 3] = 255
    ph = np.concatenate([p, np.ones((n_px, 1))], 1) @ pv.T
    depth = np.where(hit, np.clip(0.5 * ph[:, 2] / ph[:, 3] + 0.5, 0, 1), 1.0)
    return rgba.reshape(H, W, 4), depth.reshape(H, W), seg.reshape(H, W).astype(np.int32), fragile.reshape(H, W)


def linear_depth(depth, near, far, ortho=False):
    """Eye-space distance of OpenGL depth-buffer values (perspective: far*near/(far-(far-near)*d); orthographic: linear)."""
    d = np.asarray(depth, dtype=np.float64)
    return near + d * (far - near) if ortho else far * near / (far - (far - near) * d)


def compare(got, ref, near, far, ortho=False):
    """The image rule: seg agrees on >= 99.5 % of pixels; every disagreeing pixel has a non-uniform 3x3 seg neighbourhood in the
    reference; where seg agrees and the neighbourhood is uniform, linear depth is within 1e-4 z + 1e-5 m and RGB within 2 levels
    (both skipped on occlusion steps inside a uniform neighbourhood, where a ray grazes a terrain edge, and on the reference's fragile
    pixels).  Returns a message list (empty = pass)."""
    rgba, depth, seg = got
    r_rgba, r_depth, r_seg, fragile = ref
    msgs = []
    H, W = r_seg.shape
    pad = np.pad(r_seg, 1, mode="edge")
    uniform = np.ones((H, W), bool)
    zr = linear_depth(r_depth, near, far, ortho)
    # occlusion steps: a neighbour more than 10 % nearer or farther (a ray grazing a terrain edge may pass it or not)
    zpad = np.pad(zr, 1, mode="edge")
    smooth = np.ones((H, W), bool)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            uniform &= pad[1 + dy:1 + dy + H, 1 + dx:1 + dx + W] == r_seg
            smooth &= np.abs(zpad[1 + dy:1 + dy + H, 1 + dx:1 + dx + W] - zr) <= 0.1 * zr
    agree = seg == r_seg
    if agree.mean() < 0.995:
        msgs.append("seg agrees on %.4f of pixels" % agree.mean())
    bad = ~agree & uniform
    if bad.any():
        msgs.append("%d seg mismatches inside uniform neighbourhoods, first at %s (got %d, ref %d)" % (
            bad.sum(), np.argwhere(bad)[0], seg[bad][0], r_seg[bad][0]))
    cmp = agree & uniform & (r_seg >= 0)
    z = linear_depth(depth, near, far, ortho)
    dbad = cmp & smooth & ~fragile & ~(np.abs(z - zr) <= 1e-4 * zr + 1e-5)
    if dbad.any():
        msgs.append("%d depth mismatches, max |dz| %.3g" % (dbad.sum(), np.abs(z - zr)[dbad].max()))
    if (cmp & smooth).sum() < 0.5 * (r_seg >= 0).sum():
        msgs.append("only %d of %d hit pixels are compared" % ((cmp & smooth).sum(), (r_seg >= 0).sum()))
    cbad = cmp & smooth & ~fragile & (np.abs(rgba[..., :3].astype(int) - r_rgba[..., :3].astype(int)).max(-1) > 2)
    if cbad.any():
        msgs.append("%d rgb mismatches, first at %s: %s vs %s" % (cbad.sum(), np.argwhere(cbad)[0], rgba[cbad][0], r_rgba[cbad][0]))
    sky = uniform & (r_seg < 0) & agree
    if (depth[sky] != 1).any() or (rgba[sky][:, :3] != np.array(SKY)).any():
        msgs.append("sky pixels differ")
    return msgs
