// prim.h — one input element -> one output element, for the step kernel's scalar primitives.  TEST INFRASTRUCTURE ONLY.
//
// Included by the device probe (tests/gpu_probe/probe.cu, compiled by nvcc: the __CUDA_ARCH__ branches of b2q_math.cuh) and by the CPU
// emulation harness (tests/emu/emu.cpp, compiled by g++: the host branches), so both run the product's functions unchanged on the same
// element layout.  Every function reads and writes only the element it is given.
#pragma once
#include "../../paddlerobotics_b200/csrc/b2q_host_common.h"

namespace b2q_prim {
using namespace b2q;

B2Q_HD void sincos_f(float a, float* s, float* c) { m_sincos(a, *s, *c); }
B2Q_HD float rcp_f(float x) { return m_rcp(x); }
B2Q_HD float rsqrt_f(float x) { return m_rsqrt(x); }

// toe position relative to the hip joint origin p1 (what oracle.fk_leg returns), leg k's model constants
template <typename T> B2Q_HD void leg_fk(const Model<T>& md, int k, const T* q, T* out) {
  LegKin<T> K; leg_kin(md, md.leg[k], q, K);
  V3<T> r = K.toe - K.p1;
  out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
// joint angles of a foot position relative to the hip joint origin (oracle.ik_leg), leg k's signed hip offset
template <typename T> B2Q_HD void leg_inv(const Model<T>& md, int k, const T* f, T* out) {
  leg_ik(md, mk<T>(f[0], f[1], f[2]), md.leg[k].lhip, out);
}
template <typename T> B2Q_HD void rpy(const T* q, T* out) {
  V3<T> r = quat_to_rpy(q[0], q[1], q[2], q[3]);
  out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
// out = [height, nx, ny, nz]
template <typename T> B2Q_HD void terrain(const Cfg<T>& cf, T x, T y, T* out) {
  V3<T> n; out[0] = terrain_height(cf, x, y, n);
  out[1] = n.x; out[2] = n.y; out[3] = n.z;
}
// x = S^-1 b through chol6 / fwd6 / bwd6 (S packed lower, 21 entries)
template <typename T> B2Q_HD void spd_solve(const T* S21, const T* b6, T* x6) {
  T S[21], Li[6];
  for (int i = 0; i < 21; i++) S[i] = S21[i];
  for (int i = 0; i < 6; i++) x6[i] = b6[i];
  chol6(S, Li); fwd6(S, Li, x6); bwd6(S, Li, x6);
}

// the model and height-field config the step kernel builds from the default B2QConfig
template <typename T> inline Model<T> default_model() {
  B2QConfig c; default_config(&c);
  Model<T> md; build_model_host(md, c.foot_radius, c.etg_T, c.etg_amp, c.etg_phase0, c.etg_phase1, c.etg_foot_y_inset);
  return md;
}
template <typename T> inline Cfg<T> hf_cfg(int nx, int ny, double x0, double y0, double cell, const T* hf) {
  B2QConfig c; default_config(&c);
  c.terrain_type = 1; c.hf_nx = nx; c.hf_ny = ny; c.hf_x0 = x0; c.hf_y0 = y0; c.hf_cell = cell;
  return make_cfg<T>(c, hf);
}

}  // namespace b2q_prim
