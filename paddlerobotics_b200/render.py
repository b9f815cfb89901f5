"""Camera images of the GPU engine: pybullet's camera-matrix helpers, the default follow camera, and a PNG writer.

The images themselves come from the ray-cast kernel behind `b2q_render` (include/b2q_render.h), reached through
`VecQuadrupedalEnv.get_camera_image` / `QuadrupedalEnv.get_camera_image`.  Matrices are pybullet's: 16 floats, column-major
OpenGL order, as `computeViewMatrix` / `computeProjectionMatrixFOV` return them.
"""
import math
import struct
import zlib

import numpy as np

# the default follow camera (this project's own; rlschool's camera is not in the reference tree): it looks at the env's base
# from the robot's right side, slightly above
FOLLOW_OFFSET = (0.0, -1.0, 0.3)
FOLLOW_FOV, FOLLOW_NEAR, FOLLOW_FAR = 60.0, 0.1, 100.0


def _look_at_axes(eye, target, up):
    f = np.asarray(target, dtype=np.float64) - np.asarray(eye, dtype=np.float64)
    f = f / np.linalg.norm(f)
    s = np.cross(f, np.asarray(up, dtype=np.float64))
    s = s / np.linalg.norm(s)
    u = np.cross(s, f)
    return s, u, f


def compute_view_matrix(eye, target, up):
    """pybullet.computeViewMatrix(cameraEyePosition, cameraTargetPosition, cameraUpVector): gluLookAt, column-major [16]."""
    s, u, f = _look_at_axes(eye, target, up)
    e = np.asarray(eye, dtype=np.float64)
    return [float(x) for x in (s[0], u[0], -f[0], 0.0, s[1], u[1], -f[1], 0.0, s[2], u[2], -f[2], 0.0,
                               -s.dot(e), -u.dot(e), f.dot(e), 1.0)]


def compute_projection_matrix_fov(fov, aspect, near, far):
    """pybullet.computeProjectionMatrixFOV(fov [deg, vertical], aspect, nearVal, farVal): gluPerspective, column-major [16]."""
    y = 1.0 / math.tan(math.radians(fov) / 2.0)
    x = y / aspect
    nmf = near - far
    return [x, 0.0, 0.0, 0.0, 0.0, y, 0.0, 0.0, 0.0, 0.0, (far + near) / nmf, -1.0, 0.0, 0.0, 2.0 * far * near / nmf, 0.0]


def follow_camera(base_pos, width, height):
    """(view, proj) of the default follow camera for one base position."""
    t = np.asarray(base_pos, dtype=np.float64)
    return (compute_view_matrix(t + np.asarray(FOLLOW_OFFSET), t, (0.0, 0.0, 1.0)),
            compute_projection_matrix_fov(FOLLOW_FOV, width / float(height), FOLLOW_NEAR, FOLLOW_FAR))


_FOLLOW_CONSTS = {}


def follow_view_matrices(pos, out):
    """Follow-camera view matrices of many base positions on the device: pos [V,3] -> out [V,16] (float32, written in place).
    The camera's axes do not depend on the position, so only the translation column changes.  The constants are uploaded once
    per device, so later calls can be captured in a CUDA graph."""
    import torch
    key = str(out.device)
    if key not in _FOLLOW_CONSTS:
        s, u, f = _look_at_axes(FOLLOW_OFFSET, (0.0, 0.0, 0.0), (0.0, 0.0, 1.0))
        _FOLLOW_CONSTS[key] = (
            torch.tensor(np.stack([s, u, -f]).T, dtype=torch.float32, device=out.device),        # eye @ this = the rotated eye
            torch.tensor([s[0], u[0], -f[0], 0.0, s[1], u[1], -f[1], 0.0, s[2], u[2], -f[2], 0.0, 0.0, 0.0, 0.0, 1.0], dtype=torch.float32, device=out.device),
            torch.tensor(FOLLOW_OFFSET, dtype=torch.float32, device=out.device))
    rot_t, base, off = _FOLLOW_CONSTS[key]
    out.copy_(base.expand_as(out))
    out[:, 12:15] = -((pos.to(torch.float32) + off) @ rot_t)
    return out


def write_png(path, rgba):
    """rgba [H,W,4] (or [H,W,3]) uint8 -> an 8-bit PNG file, with the standard library only."""
    a = np.ascontiguousarray(np.asarray(rgba, dtype=np.uint8))
    if a.ndim != 3 or a.shape[2] not in (3, 4):
        raise ValueError("write_png: expected [H,W,4] or [H,W,3] uint8, got %s" % (a.shape,))
    h, w, c = a.shape
    raw = b"".join(b"\x00" + a[r].tobytes() for r in range(h))        # filter type 0 on every row

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    ihdr = struct.pack(">IIBBBBB", w, h, 8, 6 if c == 4 else 2, 0, 0, 0)
    with open(path, "wb") as fh:
        fh.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr) + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))
