// b2q_render.cuh — ray-cast camera images of one robot on the env's terrain (the counterpart of pybullet's getCameraImage).
// Device code shared by the sm_90a kernel (b2q_render.cu) and the CPU emulation harness (tests/emu/emu_render.cpp).
//
// One ray per pixel, all math in float32 whatever the handle's precision.  The scene of a view is 17 primitives built from
// one [37] state row with leg_kin(), the kinematics the physics uses, plus the terrain the contact test samples
// (terrain_height(): the plane z = 0 or the bilinear height field with its edge-clamped extension outside the grid).
// Conventions (pybullet / OpenGL): view and proj are column-major 4x4 matrices; the sample is the pixel centre, row 0 is the top
// row; depth is the OpenGL depth-buffer value in [0, 1] (1 = miss); segmentation ids are listed in include/b2q_render.h.
#pragma once
#include "b2q_sim.cuh"

namespace b2q {

constexpr int RENDER_NPRIM = 17;      // trunk + 4 legs x (hip, thigh, calf, toe); primitive i has segmentation id i + 1
constexpr int RENDER_TILE = 16;       // the kernel's CTA covers a 16 x 16 pixel tile
enum { RP_BOX = 0, RP_CYL = 1, RP_SPHERE = 2 };

// Collision geometry of the A1 (SURVEY App. B.3, recalled, UNVERIFIED like the inertials of b2q_model_host.h), in the engine's base
// frame (origin at the COM): full box sizes in the link frame's x, y, z.
constexpr float RG_TRUNK_X = 0.267f, RG_TRUNK_Y = 0.194f, RG_TRUNK_Z = 0.114f;
constexpr float RG_COM_OFF_X = -0.012731f, RG_COM_OFF_Y = -0.002186f, RG_COM_OFF_Z = -0.000515f;   // trunk box centre (the URDF base origin)
constexpr float RG_HIP_R = 0.046f, RG_HIP_LEN = 0.04f;                     // hip cylinder about R1.cy, centred at p1
constexpr float RG_THIGH_X = 0.034f, RG_THIGH_Y = 0.0245f, RG_THIGH_Z = 0.2f;  // thigh box in R2, centred at p2 - 0.1 R2.cz
constexpr float RG_CALF_X = 0.016f, RG_CALF_Y = 0.016f, RG_CALF_Z = 0.2f;      // calf box in R3m, centred at p3 - 0.1 R3m.cz
constexpr float RG_LINK_HALF = 0.1f;                                   // the thigh / calf box centre sits half a link length down

// Shading: Lambert from one directional light plus ambient, a fixed colour per segmentation class, a 0.25 m checkerboard on the terrain
constexpr float RS_LIGHT_X = 0.4f, RS_LIGHT_Y = -0.3f, RS_LIGHT_Z = 0.866025f;   // unit vector towards the light (|.| = 1 to 1e-6)
constexpr float RS_AMBIENT = 0.3f, RS_DIFFUSE = 0.7f, RS_CHECKER = 0.25f;
constexpr int RS_SKY_R = 178, RS_SKY_G = 204, RS_SKY_B = 230;
constexpr float RS_RIGHT_DIM = 0.8f;                        // right-side legs (0 FR, 2 RR) are drawn darker
// base colour of segmentation class `cls`: 0 trunk, 1 hip, 2 thigh, 3 calf, 4 toe, 5 / 6 the two terrain checker colours
B2Q_HD void render_colour(int cls, float* c) {
  switch (cls) {
    case 0: c[0] = 0.85f; c[1] = 0.55f; c[2] = 0.15f; break;
    case 1: c[0] = 0.35f; c[1] = 0.35f; c[2] = 0.38f; break;
    case 2: c[0] = 0.20f; c[1] = 0.40f; c[2] = 0.80f; break;
    case 3: c[0] = 0.15f; c[1] = 0.15f; c[2] = 0.18f; break;
    case 4: c[0] = 0.90f; c[1] = 0.20f; c[2] = 0.20f; break;
    case 5: c[0] = 0.70f; c[1] = 0.68f; c[2] = 0.62f; break;
    default: c[0] = 0.50f; c[1] = 0.48f; c[2] = 0.44f; break;
  }
}

struct RPrim {
  float c[3], ax[3], ay[3], az[3], h[3];   // world centre, local axes in world, half extents (cylinder: r, half length, r; sphere: r)
  int kind;
};
struct RScene {
  RPrim p[RENDER_NPRIM];
  float bc[3], br;                          // one bounding sphere around all primitives
  int robot;                                // 0: no robot in this view (non-finite state row)
};
struct RCam {
  float pv[16], inv[16];                    // proj * view and its inverse, column-major
  int ok;                                   // 0: non-finite or singular camera: every pixel is a miss
};
struct RTerrain {
  int type, nx, ny;                         // 0 plane z = 0, 1 height field [ny][nx]
  float x0, y0, icell;
  float lo, hi;                             // height range of the field: rays are clipped to this slab
};

B2Q_HD bool r_finite(float x) { return (x - x) == 0.0f; }
B2Q_HD int r_clampi(int x, int lo, int hi) { return x < lo ? lo : x > hi ? hi : x; }
// extended cell index of grid coordinate g: -1 below the grid, n - 1 at or past its last line (no int conversion of a huge float)
B2Q_HD int r_cell(float g, int n) { return g < 0.0f ? -1 : g >= (float)(n - 1) ? n - 1 : r_clampi((int)g, 0, n - 2); }

// c = a * b for column-major 4x4
B2Q_HD void r_mat4_mul(const float* a, const float* b, float* c) {
  for (int j = 0; j < 4; j++)
    for (int i = 0; i < 4; i++) {
      float s = 0.0f;
      for (int k = 0; k < 4; k++) s += a[k * 4 + i] * b[j * 4 + k];
      c[j * 4 + i] = s;
    }
}
// inverse by cofactors; false when singular or non-finite
B2Q_HD bool r_mat4_inv(const float* m, float* inv) {
  inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
  inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
  inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
  inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
  inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
  inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
  inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
  inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
  inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
  inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
  inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
  inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
  inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
  inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
  inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
  inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
  const float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
  if (!(det != 0.0f) || !r_finite(det)) return false;
  const float id = 1.0f / det;
  bool ok = true;
  for (int i = 0; i < 16; i++) { inv[i] *= id; ok = ok && r_finite(inv[i]); }
  return ok;
}
B2Q_HD void render_camera(const float* view, const float* proj, RCam& cam) {
  r_mat4_mul(proj, view, cam.pv);
  bool ok = true;
  for (int i = 0; i < 16; i++) ok = ok && r_finite(cam.pv[i]);
  cam.ok = (ok && r_mat4_inv(cam.pv, cam.inv)) ? 1 : 0;
}

B2Q_HD void r_set_prim(RPrim& p, int kind, V3<float> c, const R3<float>& Rl, float hx, float hy, float hz) {
  p.kind = kind;
  p.c[0] = c.x; p.c[1] = c.y; p.c[2] = c.z;
  p.ax[0] = Rl.cx.x; p.ax[1] = Rl.cx.y; p.ax[2] = Rl.cx.z;
  p.ay[0] = Rl.cy.x; p.ay[1] = Rl.cy.y; p.ay[2] = Rl.cy.z;
  p.az[0] = Rl.cz.x; p.az[1] = Rl.cz.y; p.az[2] = Rl.cz.z;
  p.h[0] = hx; p.h[1] = hy; p.h[2] = hz;
}
B2Q_HD R3<float> r_compose(const R3<float>& Rw, const R3<float>& Rb) {   // Rw * Rb
  R3<float> o; o.cx = rot(Rw, Rb.cx); o.cy = rot(Rw, Rb.cy); o.cz = rot(Rw, Rb.cz); return o;
}
// base pose of a [37] state row (pos3 quat4(xyzw) ...): world rotation from the normalised quaternion
B2Q_HD void render_base(const float* st, V3<float>& pos, R3<float>& R) {
  pos = mk<float>(st[0], st[1], st[2]);
  const float n = m_sqrt(st[3] * st[3] + st[4] * st[4] + st[5] * st[5] + st[6] * st[6]);
  const float in = 1.0f / n;
  R = quat_to_R<float>(st[3] * in, st[4] * in, st[5] * in, st[6] * in);
}
// the trunk box: primitive 0
B2Q_HD void render_trunk(const float* st, RPrim& p) {
  V3<float> pos; R3<float> R; render_base(st, pos, R);
  r_set_prim(p, RP_BOX, pos + rot(R, mk<float>(RG_COM_OFF_X, RG_COM_OFF_Y, RG_COM_OFF_Z)), R, 0.5f * RG_TRUNK_X, 0.5f * RG_TRUNK_Y, 0.5f * RG_TRUNK_Z);
}
// leg k's hip cylinder, thigh box, calf box and toe sphere: primitives 1 + 4k .. 4 + 4k, link frames from leg_kin()
B2Q_HD void render_leg(const Model<float>& md, int k, const float* st, RPrim* p4) {
  V3<float> pos; R3<float> R; render_base(st, pos, R);
  LegKin<float> K; leg_kin(md, md.leg[k], st + 13 + 3 * k, K);
  const R3<float> R1 = r_compose(R, K.R1), R2 = r_compose(R, K.R2), R3w = r_compose(R, K.R3m);
  r_set_prim(p4[0], RP_CYL, pos + rot(R, K.p1), R1, RG_HIP_R, 0.5f * RG_HIP_LEN, RG_HIP_R);
  r_set_prim(p4[1], RP_BOX, pos + rot(R, K.p2 - K.R2.cz * RG_LINK_HALF), R2, 0.5f * RG_THIGH_X, 0.5f * RG_THIGH_Y, 0.5f * RG_THIGH_Z);
  r_set_prim(p4[2], RP_BOX, pos + rot(R, K.p3 - K.R3m.cz * RG_LINK_HALF), R3w, 0.5f * RG_CALF_X, 0.5f * RG_CALF_Y, 0.5f * RG_CALF_Z);
  r_set_prim(p4[3], RP_SPHERE, pos + rot(R, K.toe), R3w, md.foot_r, md.foot_r, md.foot_r);
}
B2Q_HD void render_bound(RScene& sc) {
  sc.bc[0] = sc.p[0].c[0]; sc.bc[1] = sc.p[0].c[1]; sc.bc[2] = sc.p[0].c[2];
  float r = 0.0f;
  for (int i = 0; i < RENDER_NPRIM; i++) {
    const RPrim& p = sc.p[i];
    const float dx = p.c[0] - sc.bc[0], dy = p.c[1] - sc.bc[1], dz = p.c[2] - sc.bc[2];
    r = m_max(r, m_sqrt(dx * dx + dy * dy + dz * dz) + m_sqrt(p.h[0] * p.h[0] + p.h[1] * p.h[1] + p.h[2] * p.h[2]));
  }
  sc.br = r * 1.001f + 1e-4f;
}
// the whole scene of one state row, serially (the kernel builds the same primitives with one thread per leg)
B2Q_HD void render_scene(const Model<float>& md, const float* st, RScene& sc) {
  bool ok = true;
  for (int i = 0; i < 37; i++) ok = ok && r_finite(st[i]);
  sc.robot = ok ? 1 : 0;
  if (!ok) return;
  render_trunk(st, sc.p[0]);
  for (int k = 0; k < 4; k++) render_leg(md, k, st, sc.p + 1 + 4 * k);
  render_bound(sc);
}

// ---------------------------------------------------------------------------------------------------------------
// ray - primitive tests in the primitive's frame; the ray direction is a unit vector.  t of the entry point (> 0) or +inf.
B2Q_HD float r_hit_prim(const RPrim& p, V3<float> o, V3<float> d, V3<float>& nw) {
  const float inf = __builtin_huge_valf();
  const V3<float> ax = mk<float>(p.ax[0], p.ax[1], p.ax[2]), ay = mk<float>(p.ay[0], p.ay[1], p.ay[2]), az = mk<float>(p.az[0], p.az[1], p.az[2]);
  const V3<float> rel = o - mk<float>(p.c[0], p.c[1], p.c[2]);
  const V3<float> lo = mk<float>(dot(rel, ax), dot(rel, ay), dot(rel, az)), ld = mk<float>(dot(d, ax), dot(d, ay), dot(d, az));
  V3<float> nl = mk<float>(0.0f, 0.0f, 0.0f);
  float t = inf;
  if (p.kind == RP_SPHERE) {
    const float b = dot(lo, ld), c = dot(lo, lo) - p.h[0] * p.h[0], disc = b * b - c;
    if (disc >= 0.0f) {
      const float tt = -b - m_sqrt(disc);
      if (tt > 0.0f) { t = tt; nl = (lo + ld * tt) * (1.0f / p.h[0]); }
    }
  } else if (p.kind == RP_BOX) {
    float tn = -inf, tf = inf; int axis = 0; float sgn = 0.0f;
    const float o3[3] = {lo.x, lo.y, lo.z}, d3[3] = {ld.x, ld.y, ld.z};
#pragma unroll
    for (int a = 0; a < 3; a++) {
      if (d3[a] == 0.0f) {
        if (m_abs(o3[a]) > p.h[a]) tf = -inf;
        continue;
      }
      const float id = 1.0f / d3[a];
      float t0 = (-p.h[a] - o3[a]) * id, t1 = (p.h[a] - o3[a]) * id;
      const float s = d3[a] > 0.0f ? -1.0f : 1.0f;   // outward normal of the entry face
      if (t0 > t1) { const float x = t0; t0 = t1; t1 = x; }
      if (t0 > tn) { tn = t0; axis = a; sgn = s; }
      tf = m_min(tf, t1);
    }
    if (tn <= tf && tn > 0.0f) {
      t = tn;
      nl = mk<float>(axis == 0 ? sgn : 0.0f, axis == 1 ? sgn : 0.0f, axis == 2 ? sgn : 0.0f);
    }
  } else {   // cylinder about the local y axis: radius h[0], half length h[1]
    const float r = p.h[0], hl = p.h[1];
    const float a = ld.x * ld.x + ld.z * ld.z, b = lo.x * ld.x + lo.z * ld.z, c = lo.x * lo.x + lo.z * lo.z - r * r;
    if (a > 0.0f) {
      const float disc = b * b - a * c;
      if (disc >= 0.0f) {
        const float tt = (-b - m_sqrt(disc)) / a, y = lo.y + ld.y * tt;
        if (tt > 0.0f && m_abs(y) <= hl) { t = tt; nl = mk<float>((lo.x + ld.x * tt) / r, 0.0f, (lo.z + ld.z * tt) / r); }
      }
    }
    if (ld.y != 0.0f) {
      const float s = ld.y > 0.0f ? -1.0f : 1.0f;   // the cap facing the ray
      const float tt = (s * hl - lo.y) / ld.y, x = lo.x + ld.x * tt, z = lo.z + ld.z * tt;
      if (tt > 0.0f && tt < t && x * x + z * z <= r * r) { t = tt; nl = mk<float>(0.0f, s, 0.0f); }
    }
  }
  nw = ax * nl.x + ay * nl.y + az * nl.z;
  return t;
}

template <typename T>
B2Q_HD float r_hf(const T* hf, int nx, int r, int c) { return (float)hf[(size_t)r * nx + c]; }

// first crossing of the ray with the terrain for t in [0, t_end]; +inf if none.  Height field: the cells of the grid and its
// edge-clamped extension (one semi-infinite cell row / column on each side) visited in 2D-DDA order, the bilinear patch of each
// cell intersected exactly (a quadratic in t).  At most nx + ny + 2 cells, whatever the data.
template <typename T>
B2Q_HD float r_hit_terrain(const RTerrain& tr, const T* hf, V3<float> o, V3<float> d, float t_end, V3<float>& n) {
  const float inf = __builtin_huge_valf();
  n = mk<float>(0.0f, 0.0f, 1.0f);
  if (tr.type == 0) {
    if (d.z == 0.0f) return inf;
    const float t = -o.z / d.z;
    return (t >= 0.0f && t <= t_end) ? t : inf;
  }
  // the slab the heights live in (padded so that a flat field is not a zero-width slab)
  const float zlo = tr.lo - 1e-3f, zhi = tr.hi + 1e-3f;
  float t0 = 0.0f, t1 = t_end;
  if (d.z == 0.0f) {
    if (o.z < zlo || o.z > zhi) return inf;
  } else {
    const float ta = (zhi - o.z) / d.z, tb = (zlo - o.z) / d.z;
    t0 = m_max(t0, m_min(ta, tb)); t1 = m_min(t1, m_max(ta, tb));
  }
  if (!(t0 <= t1)) return inf;
  const int nx = tr.nx, ny = tr.ny;
  const float gx0 = (o.x - tr.x0) * tr.icell, gy0 = (o.y - tr.y0) * tr.icell, dgx = d.x * tr.icell, dgy = d.y * tr.icell;
  int ix = r_cell(gx0 + dgx * t0, nx), iy = r_cell(gy0 + dgy * t0, ny);
  float t = t0;
  for (int it = 0; it < nx + ny + 2; it++) {
    float tnx = inf, tny = inf;
    if (dgx > 0.0f && ix + 1 <= nx - 1) tnx = ((float)(ix + 1) - gx0) / dgx;
    else if (dgx < 0.0f && ix >= 0) tnx = ((float)ix - gx0) / dgx;
    if (dgy > 0.0f && iy + 1 <= ny - 1) tny = ((float)(iy + 1) - gy0) / dgy;
    else if (dgy < 0.0f && iy >= 0) tny = ((float)iy - gy0) / dgy;
    const float te = m_min(m_min(tnx, tny), t1);
    if (te >= t) {
      // the cell's patch: corners from clamped indices (an extension cell repeats the edge heights, so its slope terms vanish)
      const int c0 = r_clampi(ix, 0, nx - 1), c1 = r_clampi(ix + 1, 0, nx - 1), r0 = r_clampi(iy, 0, ny - 1), r1 = r_clampi(iy + 1, 0, ny - 1);
      const float h00 = r_hf(hf, nx, r0, c0), h10 = r_hf(hf, nx, r0, c1), h01 = r_hf(hf, nx, r1, c0), h11 = r_hf(hf, nx, r1, c1);
      const float a = h10 - h00, b = h01 - h00, k = h00 - h10 - h01 + h11;
      const float ue = (c0 == c1) ? 0.0f : gx0 + dgx * t - (float)ix, ve = (r0 == r1) ? 0.0f : gy0 + dgy * t - (float)iy;
      const float du = (c0 == c1) ? 0.0f : dgx, dv = (r0 == r1) ? 0.0f : dgy;
      // f(s) = z(t + s) - h(u(s), v(s)) = A s^2 + B s + C
      const float C = (o.z + d.z * t) - (h00 + a * ue + b * ve + k * ue * ve);
      const float B = d.z - (a * du + b * dv + k * (ue * dv + ve * du));
      const float A = -k * du * dv;
      const float L = te - t;
      float s = inf;
      if (C <= 0.0f) {
        s = 0.0f;
      } else if (A == 0.0f) {
        if (B < 0.0f) s = -C / B;
      } else {
        const float disc = B * B - 4.0f * A * C;
        if (disc >= 0.0f) {
          const float q = -0.5f * (B + (B >= 0.0f ? m_sqrt(disc) : -m_sqrt(disc)));
          if (q != 0.0f) {
            const float s1 = q / A, s2 = C / q;
            if (s1 >= 0.0f) s = s1;
            if (s2 >= 0.0f && s2 < s) s = s2;
          }
        }
      }
      if (s <= L) {
        const float u = m_min(m_max(ue + du * s, 0.0f), 1.0f), v = m_min(m_max(ve + dv * s, 0.0f), 1.0f);
        const float hx = (a + k * v) * tr.icell, hy = (b + k * u) * tr.icell, in = 1.0f / m_sqrt(hx * hx + hy * hy + 1.0f);
        n = mk<float>(-hx * in, -hy * in, in);
        return t + s;
      }
    }
    if (te >= t1) break;
    if (tnx <= tny) ix += dgx > 0.0f ? 1 : -1;
    else iy += dgy > 0.0f ? 1 : -1;
    t = m_max(t, te);
  }
  return inf;
}

B2Q_HD unsigned char r_u8(float x) { return (unsigned char)(m_min(m_max(x, 0.0f), 1.0f) * 255.0f + 0.5f); }

// one pixel: rgba, depth and segmentation of the ray through the centre of pixel (px, py)
template <typename T>
B2Q_HD void render_pixel(const RScene& sc, const RCam& cam, const RTerrain& tr, const T* hf, int px, int py, int W, int H,
                         unsigned char rgba[4], float& depth, int& seg) {
  rgba[0] = RS_SKY_R; rgba[1] = RS_SKY_G; rgba[2] = RS_SKY_B; rgba[3] = 255;
  depth = 1.0f; seg = -1;
  if (!cam.ok) return;
  const float xn = (2.0f * (float)px + 1.0f) / (float)W - 1.0f, yn = 1.0f - (2.0f * (float)py + 1.0f) / (float)H;
  float pn[4], pf[4];
  for (int i = 0; i < 4; i++) {
    pn[i] = cam.inv[i] * xn + cam.inv[4 + i] * yn - cam.inv[8 + i] + cam.inv[12 + i];
    pf[i] = cam.inv[i] * xn + cam.inv[4 + i] * yn + cam.inv[8 + i] + cam.inv[12 + i];
  }
  const V3<float> o = mk<float>(pn[0] / pn[3], pn[1] / pn[3], pn[2] / pn[3]);
  V3<float> d = mk<float>(pf[0] / pf[3], pf[1] / pf[3], pf[2] / pf[3]) - o;
  const float t_far = m_sqrt(dot(d, d));
  if (!(r_finite(o.x) && r_finite(o.y) && r_finite(o.z) && r_finite(t_far) && t_far > 0.0f)) return;
  d = d * (1.0f / t_far);
  float t = __builtin_huge_valf();
  V3<float> nrm = mk<float>(0.0f, 0.0f, 1.0f);
  int hit = -1;
  if (sc.robot) {
    const V3<float> rc = o - mk<float>(sc.bc[0], sc.bc[1], sc.bc[2]);
    const float b = dot(rc, d), c = dot(rc, rc) - sc.br * sc.br;
    if (b * b - c >= 0.0f && (c <= 0.0f || b < 0.0f)) {
      for (int i = 0; i < RENDER_NPRIM; i++) {
        V3<float> ni;
        const float ti = r_hit_prim(sc.p[i], o, d, ni);
        if (ti < t) { t = ti; nrm = ni; hit = i; }
      }
    }
  }
  if (t > t_far) { t = __builtin_huge_valf(); hit = -1; }
  {
    V3<float> nt;
    const float tt = r_hit_terrain<T>(tr, hf, o, d, m_min(t, t_far), nt);
    if (tt < t) { t = tt; nrm = nt; hit = RENDER_NPRIM; }
  }
  if (hit < 0) return;
  const V3<float> p = o + d * t;
  const float cz = cam.pv[2] * p.x + cam.pv[6] * p.y + cam.pv[10] * p.z + cam.pv[14];
  const float cw = cam.pv[3] * p.x + cam.pv[7] * p.y + cam.pv[11] * p.z + cam.pv[15];
  depth = m_min(m_max(0.5f * (cz / cw) + 0.5f, 0.0f), 1.0f);
  float col[3];
  if (hit == RENDER_NPRIM) {
    seg = 0;
    const float cx = floorf(p.x * (1.0f / RS_CHECKER)), cy = floorf(p.y * (1.0f / RS_CHECKER));
    render_colour(5 + (int)(cx + cy - 2.0f * floorf(0.5f * (cx + cy))), col);   // parity of the 0.25 m square
  } else {
    seg = hit + 1;
    const int cls = hit == 0 ? 0 : 1 + (hit - 1) % 4, leg = hit == 0 ? 1 : (hit - 1) / 4;
    const float dim = (leg == 0 || leg == 2) ? RS_RIGHT_DIM : 1.0f;
    render_colour(cls, col);
    col[0] *= dim; col[1] *= dim; col[2] *= dim;
  }
  const float sh = RS_AMBIENT + RS_DIFFUSE * m_max(nrm.x * RS_LIGHT_X + nrm.y * RS_LIGHT_Y + nrm.z * RS_LIGHT_Z, 0.0f);
  rgba[0] = r_u8(col[0] * sh); rgba[1] = r_u8(col[1] * sh); rgba[2] = r_u8(col[2] * sh); rgba[3] = 255;
}

}  // namespace b2q
