"""Float64 references and input sets for the step kernel's scalar primitives, shared by tests/test_emu_primitives.py (host branches, through
the CPU emulation harness) and tests/test_gpu_primitives.py (device branches, through tests/gpu_probe)."""
import numpy as np

EPS32 = float(np.finfo(np.float32).eps)
EPS64 = float(np.finfo(np.float64).eps)
TINY32 = float(np.finfo(np.float32).tiny)
L_UP, L_LOW, L_HIP = 0.2, 0.2, 0.08505
# URDF joint ranges (a1.py:186-223): hip abduction, thigh, calf
Q_LO, Q_HI = np.array([-0.802851455917, -1.0471975512, -2.69653369433]), np.array([0.802851455917, 4.18879020479, -0.916297857297])


def _dt(prec):
    return np.float64 if prec else np.float32


def ulp_err(got, ref):
    """|got - ref| in float32 ulps of ref, floored at the smallest normal's ulp (2^-149)."""
    ref = np.asarray(ref, dtype=np.float64)
    e = np.frexp(np.maximum(np.abs(ref), TINY32))[1]
    return np.abs(np.asarray(got, dtype=np.float64) - ref) / np.ldexp(1.0, e - 24)


def sign_of(leg):
    """oracle's l_hip sign of leg k (FR, FL, RR, RL): right legs -1, left legs +1."""
    return np.where(np.asarray(leg) % 2 == 1, 1, -1)


# ---- Philox4x32-10 from its published definition (Salmon et al., SC'11), vectorised over rows
def philox4x32_10(ctr, key):
    """ctr [n,4], key [n,2] uint32 -> [n,4] uint32."""
    c = [np.asarray(ctr, dtype=np.uint64)[:, i].copy() for i in range(4)]
    k0, k1 = (np.asarray(key, dtype=np.uint64)[:, i].copy() for i in range(2))
    m = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m, (k1 + np.uint64(0xBB67AE85)) & m
    return np.stack(c, 1).astype(np.uint32)


def box_muller64(words):
    """[n,4] uint32 -> [n,4] float64: philox_normal4's transform with the exact u = ((r >> 8) + 0.5) 2^-24, and the two radii [n,2]."""
    u = ((np.asarray(words, dtype=np.uint64) >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    ra, rb = np.sqrt(-2 * np.log(u[:, 0])), np.sqrt(-2 * np.log(u[:, 2]))
    tp = 2 * np.pi
    return np.stack([ra * np.cos(tp * u[:, 1]), ra * np.sin(tp * u[:, 1]), rb * np.cos(tp * u[:, 3]), rb * np.sin(tp * u[:, 3])], 1), np.stack([ra, rb], 1)


def philox_inputs(n, seed=0):
    """n (seed, counter) tuples: random keys, a quarter with the high key word zero, and counters at 0 and 2^32 - 1."""
    rng = np.random.default_rng(seed)
    key = rng.integers(0, 2 ** 32, (n, 2), dtype=np.uint64)
    key[::4, 1] = 0
    ctr = rng.integers(0, 2 ** 32, (n, 3), dtype=np.uint64)
    ctr[1::8] = 0
    ctr[5::8] = 0xFFFFFFFF
    seeds = (key[:, 1] << np.uint64(32)) | key[:, 0]
    return seeds.astype(np.uint64), ctr.astype(np.uint32), key.astype(np.uint32)


# ---- leg kinematics
def fk_grid(m):
    """[4 m^3, 3] joint angles on an m x m x m grid over the URDF ranges, and the leg of each row."""
    g = [np.linspace(Q_LO[j], Q_HI[j], m) for j in range(3)]
    q = np.stack(np.meshgrid(*g, indexing="ij"), -1).reshape(-1, 3)
    return np.tile(q, (4, 1)), np.repeat(np.arange(4), q.shape[0])


def fk_ref(q, legs):
    from oracle import oracle as O
    return np.array([O.fk_leg(q[i], int(sign_of(legs[i]))) for i in range(len(legs))])


def ik_ref(f, legs):
    from oracle import oracle as O
    return np.array([O.ik_leg(f[i], int(sign_of(legs[i]))) for i in range(len(legs))])


def ik_inputs(n, seed=0):
    """[n,3] foot positions relative to the hip joint origin and their legs: a third uniform in the reachable shell, a third within 1e-6
    of its outer boundary |f|^2 = l_hip^2 + (l_up + l_low)^2 (both sides), a third near its inner limit y^2 + z^2 = l_hip^2 (the foot on
    the hip's axis cylinder) and the knee folded back onto the thigh."""
    rng = np.random.default_rng(seed)
    legs = rng.integers(0, 4, n)
    k = n // 3
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    rmax = np.sqrt(L_HIP ** 2 + (L_UP + L_LOW) ** 2)
    r = np.empty(n)
    r[:k] = rng.uniform(0.05, rmax, k)
    r[k:2 * k] = rmax * (1 + rng.uniform(-1e-6, 1e-6, k))
    f = d * r[:, None]
    # inner limit: y^2 + z^2 = l_hip^2 (1 + eps) with x free inside the shell
    m = n - 2 * k
    phi = rng.uniform(-np.pi, np.pi, m)
    rho = L_HIP * np.sqrt(1 + rng.uniform(-1e-5, 1e-5, m))
    f[2 * k:, 0] = rng.uniform(-0.35, 0.35, m)
    f[2 * k:, 1], f[2 * k:, 2] = rho * np.cos(phi), rho * np.sin(phi)
    return f, legs


def ik_margins(f, legs):
    """float64 distance of leg_ik's acos and asin arguments from the edge of [-1, 1] (negative: outside, the IK is NaN)."""
    lh = L_HIP * sign_of(legs)
    x, y, z = f[:, 0], f[:, 1], f[:, 2]
    ca = (x * x + y * y + z * z - lh * lh - L_LOW ** 2 - L_UP ** 2) / (2 * L_LOW * L_UP)
    with np.errstate(invalid="ignore"):
        tk = -np.arccos(np.clip(ca, -1, 1))
        l = np.sqrt(L_UP ** 2 + L_LOW ** 2 + 2 * L_UP * L_LOW * np.cos(tk))
        sa = -x / l
    return np.minimum(1 - np.abs(ca), 1 - np.abs(sa))


# ---- quat_to_rpy
def quat_inputs(n, seed=0):
    """[n,4] xyzw unit quaternions: uniform, a band within 1e-3 of pitch = +-pi/2, and yaw / roll at the +-pi branch cut."""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 4))
    k = n // 4
    r, p, y = rng.uniform(-np.pi, np.pi, k), rng.choice([-1, 1], k) * (np.pi / 2 - 10 ** rng.uniform(-8, -3, k)), rng.uniform(-np.pi, np.pi, k)
    q[:k] = rpy_to_quat(r, p, y)
    cut = np.pi * rng.choice([-1, 1], k) * (1 - rng.uniform(0, 1e-6, k))
    q[k:2 * k] = rpy_to_quat(rng.uniform(-1, 1, k), rng.uniform(-1, 1, k), cut)
    q[2 * k:3 * k] = rpy_to_quat(cut, rng.uniform(-1, 1, k), rng.uniform(-1, 1, k))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def rpy_to_quat(r, p, y):
    cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2), np.sin(y / 2)
    return np.stack([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy], -1)


def rpy_to_R(a):
    """R = Rz(yaw) Ry(pitch) Rx(roll), [n,3,3]."""
    r, p, y = a[:, 0], a[:, 1], a[:, 2]
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    return np.stack([np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr], -1),
                     np.stack([sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr], -1),
                     np.stack([-sp, cp * sr, cp * cr], -1)], 1)


def quat_to_R(q):
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)


def rpy_ref(q):
    from oracle import oracle as O
    return np.array([O.quat_to_rpy(qq) for qq in q])


def angle_diff(a, b):
    return np.abs((a - b + np.pi) % (2 * np.pi) - np.pi)


# ---- terrain
FIELDS = [  # (ny, nx, x0, y0, cell): both sides of the 17-cell boundary, non-square, negative origins
    (5, 9, -0.3, -0.2, 0.05), (16, 16, -0.4, -0.4, 0.05), (17, 17, 0.0, 0.0, 0.05), (24, 40, -1.0, -0.6, 0.05), (40, 24, -1.25, 0.5, 0.03), (2, 2, -0.1, -0.1, 0.2)]


def terrain_points(ny, nx, x0, y0, cell, rng, n=2000):
    """Every cell corner, the midpoint of every cell edge, points 0.5 to 3 cells beyond every edge and corner of the field, random interior."""
    gx, gy = np.meshgrid(np.arange(nx), np.arange(ny))
    corners = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.float64)
    edges = np.concatenate([corners + [0.5, 0], corners + [0, 0.5]])
    t = rng.uniform(0, 1, (n, 2)) * [nx - 1, ny - 1]
    out = rng.uniform(0.5, 3, (n, 2)) * rng.choice([-1, 1], (n, 2))
    far = np.where(out > 0, out + [nx - 1, ny - 1], out)
    mixed = far.copy(); mixed[: n // 2, 0] = t[: n // 2, 0]; mixed[n // 2:, 1] = t[n // 2:, 1]
    g = np.concatenate([corners, edges, t, far, mixed])
    return np.stack([x0 + g[:, 0] * cell, y0 + g[:, 1] * cell], 1)


def terrain_ref(hf, x0, y0, cell, xy, top=1.000001, cells32=False):
    """[n,4] (height, normal) of terrain_height in float64: the bilinear patch at the clamped point (far edges at n - top, as the kernel
    and the oracle clamp) and that patch's analytic gradient; tests/render_ref.hf_height is the same with top = 1.  The normal jumps at
    cell edges, so for a float32 kernel `cells32` takes the clamped cell coordinates as float32 computes them and the rest in float64."""
    ny, nx = hf.shape
    if cells32:
        f = np.float32
        fx = np.minimum(np.maximum((f(xy[:, 0]) - f(x0)) * f(1.0 / cell), f(0)), f(nx) - f(top)).astype(np.float64)
        fy = np.minimum(np.maximum((f(xy[:, 1]) - f(y0)) * f(1.0 / cell), f(0)), f(ny) - f(top)).astype(np.float64)
    else:
        fx = np.minimum(np.maximum((xy[:, 0] - x0) * (1.0 / cell), 0.0), nx - top)
        fy = np.minimum(np.maximum((xy[:, 1] - y0) * (1.0 / cell), 0.0), ny - top)
    ix, iy = np.minimum(fx.astype(np.int64), nx - 2), np.minimum(fy.astype(np.int64), ny - 2)
    tx, ty = fx - ix, fy - iy
    h00, h10, h01, h11 = hf[iy, ix], hf[iy, ix + 1], hf[iy + 1, ix], hf[iy + 1, ix + 1]
    h = (1 - tx) * (1 - ty) * h00 + tx * (1 - ty) * h10 + (1 - tx) * ty * h01 + tx * ty * h11
    hx = ((1 - ty) * (h10 - h00) + ty * (h11 - h01)) / cell
    hy = ((1 - tx) * (h01 - h00) + tx * (h11 - h10)) / cell
    n = np.stack([-hx, -hy, np.ones_like(hx)], 1)
    return np.concatenate([h[:, None], n / np.linalg.norm(n, axis=1, keepdims=True)], 1)


# ---- 6x6 SPD solves
TRI = [(i, j) for i in range(6) for j in range(i + 1)]          # packed lower order of b2q_math.cuh's tri(i, j)


def pack21(S):
    return np.stack([S[:, i, j] for i, j in TRI], 1)


def spd_set(n_per, conds, seed=0):
    """[m,6,6] SPD matrices Q diag(geomspace(1, 1/kappa)) Q^T for each condition number kappa, with their kappas."""
    rng = np.random.default_rng(seed)
    mats, ks = [], []
    for k in conds:
        for _ in range(n_per):
            Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
            s = np.geomspace(1.0, 1.0 / k, 6) * 10 ** rng.uniform(-2, 2)
            mats.append((Q * s) @ Q.T); ks.append(k)
    S = np.array(mats)
    return 0.5 * (S + S.transpose(0, 2, 1)), np.array(ks, dtype=np.float64)


def schur_set():
    """The base's 6x6 articulated inertia S = H_bb - H_bq H_qq^-1 H_qb of the oracle's mass matrix at the reset pose, over the full-range
    dynamics rows that scale masses and inertias (tests/full_range.py) and the seeded draws."""
    from oracle import oracle as O
    import full_range as FR
    rows = list(FR._corners().values()) + list(FR.drawn_rows().values())
    out = []
    for r in rows:
        o = O.OracleEnv(O.default_config(), r, settle=False)
        o.reset()
        M = o.mass_matrix()
        S = M[:6, :6] - M[:6, 6:] @ np.linalg.solve(M[6:, 6:], M[6:, :6])
        out.append(0.5 * (S + S.T))
    S = np.array(out)
    return S, np.linalg.cond(S)


# ---- checks shared by the host (tests/emu/emu.py) and device (tests/gpu_probe/probe.py) backends; each returns its measured maxima
def check_kinematics(be, prec, m=16, n_ik=6000):
    """leg_kin against oracle.fk_leg on an m^3 grid per leg, leg_ik against oracle.ik_leg on ik_inputs.  NaN classification: where
    ik_margins > c eps32 float32 must be finite, where < -c eps32 it must be NaN; in between either is accepted (inside the calf's URDF range).  Returns the errors, the
    largest |margin| / eps32 at which float32 and float64 disagree about NaN, and the number of classification violations at c = 128
    (disagreements measured within 3.3 eps32 on the host and on H100)."""
    q, legs = fk_grid(m)
    fk = be.leg(prec, legs, q, False)
    fk_err = float(np.max(np.abs(fk - fk_ref(q, legs))))
    f, fl = ik_inputs(n_ik)
    ik = be.leg(prec, fl, f, True).astype(np.float64)
    ref = ik_ref(f.astype(_dt(prec)).astype(np.float64), fl)
    marg = ik_margins(f.astype(_dt(prec)).astype(np.float64), fl)
    fin_k, fin_r = np.isfinite(ik).all(1), np.isfinite(ref).all(1)
    both = fin_k & fin_r
    err = np.max(np.abs(ik - ref), axis=1)
    eps = EPS32 if prec == 0 else EPS64
    c = 128
    # past the URDF calf range (|knee| > 2.7, the knee folding onto the thigh) l -> 0 and asin(-x / l) is ill-conditioned: left out
    with np.errstate(invalid="ignore"):
        knee_ok = ~(np.arccos(np.clip((np.sum(f * f, 1) - L_HIP ** 2 - L_LOW ** 2 - L_UP ** 2) / (2 * L_LOW * L_UP), -1, 1)) > -Q_LO[2])
    viol = int(np.sum(knee_ok & (marg > c * eps) & ~fin_k) + np.sum(knee_ok & (marg < -c * eps) & fin_k))
    dis = knee_ok & (fin_k != fin_r)
    return {"fk": fk_err, "ik_interior": float(err[both & (marg > 1e-3)].max()), "ik_boundary": float(err[both & (marg <= 1e-3)].max(initial=0)),
            "nan_disagree_max_margin_eps": float(np.abs(marg[dis]).max(initial=0) / eps), "nan_violations": viol,
            "n_boundary": int(np.sum(both & (marg <= 1e-3))), "n_nan": int(np.sum(~fin_r))}


def check_rpy(be, prec, n=40000):
    """quat_to_rpy against oracle.quat_to_rpy on the same (rounded) quaternions: angles mod 2 pi away from the gimbal band, and inside it
    (|pitch| within 1e-3 of pi/2, where roll and yaw are not determined individually) the rotations rebuilt from the two angle triples,
    in units of eps / cos(pitch): the atan2 arguments of roll and yaw shrink with cos(pitch) while their rounding does not, so within
    ~eps of the pole roll and yaw are rounding alone (getEulerFromQuaternion's formula, in the oracle as in the kernel)."""
    q = quat_inputs(n).astype(_dt(prec))
    got = be.rpy(prec, q).astype(np.float64)
    qd = q.astype(np.float64)
    ref = rpy_ref(qd)
    gim = np.abs(np.abs(ref[:, 1]) - np.pi / 2) < 1e-3
    ang = angle_diff(got, ref).max(1)
    rot = np.abs(rpy_to_R(got) - rpy_to_R(ref)).max((1, 2))
    eps = EPS32 if prec == 0 else EPS64
    scaled = rot * np.maximum(np.cos(ref[:, 1]), eps) / eps              # rounding of the atan2 arguments, relative to cos(pitch)
    return {"angles": float(ang[~gim].max()), "gimbal_rotation_scaled": float(scaled[gim].max()), "rotation": float(rot[~gim].max()),
            "pitch_in_gimbal": float(angle_diff(got[gim, 1], ref[gim, 1]).max()), "n_gimbal": int(gim.sum())}


def check_terrain(be, prec, seed=0):
    """terrain_height and its normal on every field of FIELDS against terrain_ref (the kernel's clamp); the height also against
    render_ref.hf_height, whose clamp at n - 1 differs by at most 1e-6 of a cell's rise.  A NaN coordinate gives the height at the clamped
    near edge (fmax(NaN, 0) = 0)."""
    import render_ref
    rng = np.random.default_rng(seed)
    out = {"height": 0.0, "normal": 0.0, "vs_hf_height": 0.0}
    for ny, nx, x0, y0, cell in FIELDS:
        hf = rng.uniform(-0.3, 0.3, (ny, nx))
        xy = terrain_points(ny, nx, x0, y0, cell, rng).astype(_dt(prec))
        got = be.terrain(prec, hf, x0, y0, cell, xy).astype(np.float64)
        ref = terrain_ref(hf, x0, y0, cell, xy.astype(np.float64), cells32=prec == 0)
        hh = render_ref.hf_height(hf, x0, y0, cell, xy[:, 0].astype(np.float64), xy[:, 1].astype(np.float64))
        assert np.isfinite(got).all()
        out["height"] = max(out["height"], float(np.abs(got[:, 0] - ref[:, 0]).max()))
        out["normal"] = max(out["normal"], float(np.abs(got[:, 1:] - ref[:, 1:]).max()))
        out["vs_hf_height"] = max(out["vs_hf_height"], float(np.abs(got[:, 0] - hh).max()))
        nan = be.terrain(prec, hf, x0, y0, cell, np.array([[np.nan, y0 + 0.5 * cell], [x0 + 0.5 * cell, np.nan], [np.nan, np.nan]], dtype=_dt(prec)))
        edge = terrain_ref(hf, x0, y0, cell, np.array([[x0, y0 + 0.5 * cell], [x0 + 0.5 * cell, y0], [x0, y0]]))
        assert np.allclose(nan.astype(np.float64), edge, rtol=0, atol=1e-6 if prec == 0 else 1e-15), (nan, edge)
    return out


def check_solve(be, prec):
    """chol6 / fwd6 / bwd6 solve error ||x - x*|| / ||x*|| over kappa eps, for SPD matrices of condition 10 .. 1e6 and the oracle's
    Schur complements, the solve in float32 or float64 from the matrix rounded to that precision."""
    eps = EPS32 if prec == 0 else EPS64
    S1, k1 = spd_set(200, [1e1, 1e2, 1e3, 1e4, 1e5, 1e6])
    S2, k2 = schur_set()
    res = {}
    for name, S, k in (("synthetic", S1, k1), ("schur", S2, k2)):
        rng = np.random.default_rng(1)
        St = S.astype(_dt(prec)).astype(np.float64)
        x_true = rng.normal(size=(S.shape[0], 6))
        b = np.einsum("nij,nj->ni", St, x_true).astype(_dt(prec))
        xs = np.linalg.solve(St, b.astype(np.float64)[..., None])[..., 0]       # the exact solution of the rounded system
        got = be.solve(prec, pack21(St), b).astype(np.float64)
        kk = np.linalg.cond(St)
        rel = np.linalg.norm(got - xs, axis=1) / np.linalg.norm(xs, axis=1)
        res[name] = float(np.max(rel / (kk * eps)))
        res[name + "_max_cond"] = float(kk.max())
    return res
